"""CPU tests of the PRODUCT's kernel logic: the __host__ __device__ phase functions that the sm_90a
kernels execute (microwakeword_b200/csrc/*_dev.cuh) are run thread-by-thread on the host
(tests/host_emul) and compared with the oracle.  This is what lets index math and bit-exactness be
iterated without a GPU; the GPU runs of the very same functions are in tests/test_gpu_parity.py."""

import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN, edge_case_audio, synth_audio
from host_emul import emul
from microwakeword_b200 import model_file as MF


def test_product_tables_equal_oracle_tables():
    t, o = emul.tables(), oracle.Frontend().tables()
    for k in ("window", "bin_weight", "bin_unweight", "chan_start", "gain_lut", "log_lut", "twiddles", "super_twiddles"):
        assert np.array_equal(t[k], o[k]), k
    assert t["info"][0] == 5 and t["info"][1] == 241 and t["info"][2] == 1
    assert t["info"][3] == 800            # span coefficients: int32 [slot][lane][stride] copy in shared memory
    assert sum(t["info"][4:8]) <= 48      # per-lane trip count of the balanced filterbank schedule


def test_isqrt_matches_library_rule():
    L, O = emul.lib(), oracle.lib()
    rng = np.random.default_rng(0)
    vals = [0, 1, 2, 3, (1 << 32) - 1, 1 << 32, (1 << 64) - 1, 1 << 63, 65535 ** 2 + 65535, 65535 ** 2 + 65536,
            (2 ** 32 - 1) ** 2, (2 ** 32 - 1) ** 2 + 2 ** 32 - 1, (2 ** 32 - 1) ** 2 + 2 ** 32]
    vals += [int(v) for v in rng.integers(0, 1 << 62, 5000)] + [int(v) for v in rng.integers(0, 1 << 36, 5000)]
    vals += [int(r) * int(r) + int(r) + int(d) for r, d in zip(rng.integers(1, 1 << 31, 5000), rng.integers(-2, 3, 5000))]
    for v in vals:
        assert L.emul_isqrt64_round(v) == O.mwwo_sqrt64(v), v
        assert L.emul_isqrt64_round_fast(v) == O.mwwo_sqrt64(v), v


def test_isqrt_fp64_fast_path_is_exact_below_2_48():
    """K1 takes one IEEE double sqrt for accumulators < 2^48 (mww_frontend_dev.cuh::isqrt64_round_fast).  The only
    inputs that could break trunc(RN(sqrt x) + 0.5) sit next to a half-integer root: x = n^2 - n and n^2 - n + 1;
    sweep them densely up to n = 2^24 together with squares, the 32/64-bit seam of the library and random values."""
    L, O = emul.lib(), oracle.lib()
    rng = np.random.default_rng(1)
    n = np.concatenate([np.arange(1, 1 << 16, dtype=np.uint64), rng.integers(1 << 16, 1 << 24, 1 << 20).astype(np.uint64),
                        np.arange((1 << 24) - 4096, 1 << 24, dtype=np.uint64)])
    cand = np.concatenate([n * n - n, n * n - n + 1, n * n, n * n + n, n * n + n + 1, n * n - 1,
                           rng.integers(0, 1 << 48, 1 << 20).astype(np.uint64), rng.integers(0, 1 << 33, 1 << 18).astype(np.uint64),
                           np.arange((1 << 32) - 70000, (1 << 32) + 70000, dtype=np.uint64),
                           (np.uint64(1) << np.uint64(48)) - np.arange(1, 4096, dtype=np.uint64)])
    cand = np.ascontiguousarray(cand[cand < (1 << 48)])
    assert L.emul_isqrt_fast_mismatch(cand.ctypes.data, cand.size) == -1
    for v in (0, 1, 2, 65535 ** 2 + 65535, 65535 ** 2 + 65536, (1 << 32) - 1, 1 << 32, (1 << 48) - 1, 1 << 48, (1 << 64) - 1):
        assert L.emul_isqrt64_round_fast(v) == O.mwwo_sqrt64(v), v


def test_frontend_phases_bit_exact_random_edge_and_adversarial():
    rng = np.random.default_rng(0)
    n = 3200
    t = np.arange(n)
    rows = [synth_audio(n, 40 + i) for i in range(12)] + list(edge_case_audio(n))
    for i in range(120):                     # full-scale patterns that overflow int16 inside the FFT butterflies
        kind = i % 4
        if kind == 0:
            x = rng.choice([-32768, 32767], n)
        elif kind == 1:
            x = rng.integers(-32768, 32768, n)
        elif kind == 2:
            w = rng.choice([np.pi / 2, np.pi / 4, np.pi / 8, 3 * np.pi / 8, rng.uniform(0, np.pi)])
            x = 32767 * np.sign(np.cos(w * (t // 2) + rng.uniform(0, 6.28) + (t % 2) * np.pi / 2) + 1e-12)
        else:
            x = np.clip(rng.normal(0, 30000, n), -32768, 32767)
        rows.append(np.clip(np.round(x), -32768, 32767).astype(np.int16))
    audio = np.stack(rows)
    got = emul.Frontend(audio.shape[0]).features(audio)
    want, _ = oracle.run_pipeline(None, audio, want_probs=False)
    assert got.shape == want.shape and np.array_equal(got, want)


def test_filterbank_schedule_is_bank_conflict_free_and_complete():
    """The per-lane energy loads of the mel accumulation are where K1's shared-memory bank conflicts would sit.  The
    table builder picks even start words whose (word / 2) mod 16 is a permutation over the 16 lanes of a slot, so each
    64-bit load of a half-warp (= one frame) covers the 32 banks exactly once -- for the energies and for the int32 coefficient rows; and the shifted / padded spans still reproduce the
    triangular weights of every channel."""
    slots, coef = emul.fb_schedule()
    t = emul.tables()
    lens = [int(v) for v in t["info"][4:8]]
    assert lens == [28, 12, 6, 0]
    seen_channels = set()
    for s, L in enumerate(lens):
        if L == 0:
            continue
        for j in range(0, L, 2):                                  # the j-th 64-bit load of the slot
            e_words = slots[:, s, 1].astype(int) + j
            c_words = slots[:, s, 3].astype(int) + j
            for words in (e_words, c_words):
                assert np.all(words % 2 == 0)
                assert sorted((words // 2) % 16) == list(range(16)), (s, j)
        for lane in range(16):
            ch, word0, n, off = (int(v) for v in slots[lane, s])
            assert 0 <= word0 and word0 + L <= 272 and 0 <= off and off + L <= 800
            row = coef[off:off + L]
            if ch < 0:
                assert not row.any()
                continue
            seen_channels.add(ch)
            # row position w holds the coefficient of FFT bin word0 + w - 1 (energy of bin k lives at word k + 1)
            b0, b1, b2 = (int(t["chan_start"][ch + i]) for i in range(3))
            want = np.zeros(L, np.int64)
            for b in range(b0, b2):
                want[b + 1 - word0] = t["bin_unweight"][b] if b < b1 else t["bin_weight"][b]
            assert np.array_equal(row, want), (lane, s, ch)
    assert seen_channels == set(range(40))


def test_filterbank_accumulators_stay_below_2_48():
    """k1_filterbank takes the FP64 square root, exact below 2^48, for every channel; a warp vote sends accumulators >= 2^48
    to the integer routine.  Bound every accumulator from the product's tables: each real-FFT half out of k1_real_energy is
    (f1 +- t) >> 1 with f1 the sum of two C_FIXDIV(., 2) of int16 values and t an int16, so every energy is at most
    2 * max|half|^2, and an accumulator is at most that times the sum of its slot's coefficients.  Below 2^48 the vote
    cannot fire for any int16 or float audio."""
    i16 = np.arange(-32768, 32768, dtype=np.int64)
    fixdiv2 = (i16 * 16383 + 16384) >> 15
    f1 = (2 * int(fixdiv2.min()), 2 * int(fixdiv2.max()))
    # (f1 + t) >> 1, (f1 - t) >> 1 and (t - f1) >> 1 are monotone in f1 and t: the extremes sit at the corners
    halves = [(a + s * t) >> 1 for a in f1 for t in (-32768, 32767) for s in (1, -1)] + [(t - a) >> 1 for a in f1 for t in (-32768, 32767)]
    half = max(abs(h) for h in halves)
    assert half == 32767
    energy = 2 * half * half
    assert energy < 1 << 31                              # also below the int32 view the accumulation widens from
    slots, coef = emul.fb_schedule()
    lens = [int(v) for v in emul.tables()["info"][4:8]]
    worst = 0
    for lane in range(16):
        for s, L in enumerate(lens):
            ch, _, _, off = (int(v) for v in slots[lane, s])
            if L == 0:
                continue
            row = coef[off:off + L].astype(np.int64)
            assert (row >= 0).all()
            worst = max(worst, int(row.sum()) * energy)
            assert ch >= 0 or not row.any()
    assert 0 < worst < 1 << 48, worst
    assert worst < 1 << 47                              # 1.22e14 (coefficient sum 56 902): a factor two to spare


def test_fused_clip_frontend_phases_bit_exact_and_order_independent():
    """The one-launch clip frontend (filterbank -> estimate recurrence on 40 threads -> 640 independent outputs per group,
    all from shared memory) against the oracle: multi-group calls, a ragged last group, chunked feeding with carried state,
    and ascending vs descending thread order inside every phase (an intra-phase race would make them differ)."""
    rng = np.random.default_rng(3)
    rows = [synth_audio(16000, 170 + i) for i in range(4)] + [e[:16000] for e in edge_case_audio(16000)[:6]]
    rows.append(rng.choice([-32768, 32767], 16000).astype(np.int16))
    audio = np.stack(rows)
    want, _ = oracle.run_pipeline(None, audio, want_probs=False)
    for order in (0, 1):
        got = emul.Frontend(audio.shape[0]).features(audio, fused=True, order=order)       # 98 frames: 6 groups + 2 frames
        assert got.shape == want.shape and np.array_equal(got, want), order
    fe, sep = emul.Frontend(audio.shape[0]), emul.Frontend(audio.shape[0])
    pos, parts = 0, []
    for n in (4000, 1760, 6400, 3840):                                # fused and separate phases interleave on one state
        fused = len(parts) % 2 == 0
        parts.append(fe.features(audio[:, pos:pos + n], fused=fused))
        sep.features(audio[:, pos:pos + n])
        assert np.array_equal(fe.estimate, sep.estimate) and np.array_equal(fe.carry, sep.carry)
        pos += n
    assert np.array_equal(np.concatenate(parts, 1), want)


@pytest.mark.parametrize("step_ms", [20, 30, 7, 25, 1])
def test_run_time_window_step_phases_bit_exact(step_ms):
    """window_step != 10 ms (audio_utils.py:69-81, default 20): groups of fewer than 16 frames when the hop is long, frames
    overlapping heavily when it is short, leftover samples carried between odd-sized chunks -- against the oracle frontend
    built with that step."""
    hop = 16 * step_ms
    audio = np.stack([synth_audio(9000, 310 + i) for i in range(2)] + [edge_case_audio(9000)[1]])
    want = []
    for row in audio:
        fe = oracle.Frontend((16000, 30, step_ms, 40, 125.0, 7500.0))
        fe.reset()
        want.append(fe.stream(row))
    want = np.stack(want)
    got = emul.Frontend(3).features(audio, hop=hop)
    assert got.shape == want.shape and np.array_equal(got, want)
    fe, pos, parts = emul.Frontend(3), 0, []
    for n in (2000, 16, 1234, 3750, 2000):
        parts.append(fe.features(audio[:, pos:pos + n], hop=hop))
        pos += n
    assert np.array_equal(np.concatenate(parts, 1), want)


def test_frontend_phases_chunked_stream_and_multi_group():
    audio = np.stack([synth_audio(16000, 70 + i) for i in range(3)])     # 98 frames -> 7 groups of 16
    want, _ = oracle.run_pipeline(None, audio, want_probs=False)
    fe = emul.Frontend(3)
    rng = np.random.default_rng(1)
    pos, parts = 0, []
    while pos < audio.shape[1]:
        n = int(rng.integers(1, 2500))
        parts.append(fe.features(audio[:, pos:pos + n]))
        pos += n
    assert np.array_equal(np.concatenate(parts, 1), want)
    assert fe.used == 320


def test_nn_f32_phases_match_oracle_and_golden():
    t = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    feats = np.load(os.path.join(GOLDEN, "config0_features.npy"))
    want = np.load(os.path.join(GOLDEN, "config0_probs_f32.npy"))
    nn = emul.NnF32(t, 1)
    got = nn.infer(feats[None, :996])                 # 332 steps = 10 full chunks of 32 + a ragged one
    assert got.shape == (1, 332) and np.abs(got[0] - want).max() <= 1e-5
    # ragged calls leave pending rows; the chain continues exactly
    nn = emul.NnF32(t, 1)
    parts = [nn.infer(feats[None, a:b]) for a, b in ((0, 1), (1, 5), (5, 100), (100, 101), (101, 997))]
    assert np.array_equal(np.concatenate(parts, 1), got)
    # float32 rows == uint16 rows * 0.0390625
    nn = emul.NnF32(t, 1)
    assert np.array_equal(nn.infer((feats[None, :996].astype(np.float32) * np.float32(0.0390625))), got)


def test_nn_int8_phases_bit_exact():
    q = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"))
    feats = np.load(os.path.join(GOLDEN, "batch_features.npy"))
    want = np.load(os.path.join(GOLDEN, "batch_probs_int8.npy"))
    nn = emul.NnI8(q, feats.shape[0])
    assert np.array_equal(nn.infer(feats), want)
    f0 = np.load(os.path.join(GOLDEN, "config0_features.npy"))
    nn = emul.NnI8(q, 1)
    parts = [nn.infer(f0[None, a:b]) for a, b in ((0, 2), (2, 300), (300, 301), (301, 997))]
    assert np.array_equal(np.concatenate(parts, 1)[0], np.load(os.path.join(GOLDEN, "config0_probs_int8.npy")))


def test_wgmma_operand_layout_round_trips_and_is_a_swizzle_bijection():
    """The wgmma clip kernel's shared-memory operand layout (mww_nn_tc_prep.h; GPU parity proves the kernel, this pins the
    layout on the CPU): within a K-slot [rows][128 B] the swizzle permutes the eight 16-byte chunks of a row by (row & 7) --
    a bijection onto the slot, a row stays 128 contiguous bytes (the conflict-free store the kernel relies on); the weight
    planes read back through the same map give hi + lo == w exactly, hi is a TF32 (13 low mantissa bits clear), |lo| <= 2^-10 |w|,
    and the tail of the last slot is zero."""
    import ctypes
    L = emul.lib()
    L.emul_sw128_off.restype = ctypes.c_uint
    L.emul_tc_layout.restype = ctypes.c_longlong
    for rows in (32, 64, 128):
        off = np.array([[L.emul_sw128_off(r, kk) for kk in range(32)] for r in range(rows)], np.int64)
        assert np.array_equal(np.sort(off.ravel()), 4 * np.arange(rows * 32))                       # bijection onto the slot, 4-byte aligned
        assert all(np.array_equal(np.sort(off[r]), r * 128 + 4 * np.arange(32)) for r in range(rows))   # a row = 128 contiguous bytes
        chunk = (off % 128) // 16
        assert np.array_equal(chunk, (np.arange(32)[None, :] // 4) ^ (np.arange(rows)[:, None] & 7))      # the hardware's 128-byte XOR swizzle
    rng = np.random.default_rng(3)
    for K, N in ((200, 32), (32, 64), (64, 64)):
        w = (rng.standard_normal((K, N)) * rng.choice([1e-3, 1.0, 50.0], (K, N))).astype(np.float32)
        n = L.emul_tc_layout(w.ctypes.data_as(ctypes.c_void_p), K, N, None, 0)
        slots, plane = (K + 31) // 32, N * 128
        assert n == slots * 2 * plane
        blob = np.zeros(n, np.uint8)
        L.emul_tc_layout(w.ctypes.data_as(ctypes.c_void_p), K, N, blob.ctypes.data_as(ctypes.c_void_p), ctypes.c_longlong(n))
        f = blob.view(np.float32)
        hi, lo = np.zeros((slots * 32, N), np.float32), np.zeros((slots * 32, N), np.float32)
        for k in range(slots * 32):
            for col in range(N):
                o = (k // 32) * 2 * plane + L.emul_sw128_off(col, k % 32)
                hi[k, col], lo[k, col] = f[o // 4], f[(o + plane) // 4]
        assert np.array_equal(hi[:K] + lo[:K], w) and not hi[K:].any() and not lo[K:].any()
        assert not (hi.view(np.uint32) & 0x1FFF).any()
        assert (np.abs(lo[:K]) <= np.abs(w) * 2.0 ** -10).all()


def test_feature_quantisation_table_is_the_reference_expression_for_every_uint16():
    """NnWeightsI8::qlut (built by mww_create and by the emulation with build_feature_qlut): every one of the 65 536 possible
    uint16 features maps to what Model.quantize_input_data computes for feature * 0.0390625 (inference.py:93-94, 127-147)."""
    import ctypes
    from oracle import mixednet_ref as R
    u = np.arange(65536, dtype=np.uint16)
    x = u.astype(np.float32) * np.float32(0.0390625)
    for scale, zp in ((0.10196078568696976, -128), (0.0390625, -128), (0.25, 3), (1.0 / 3.0, -7), (26.0, 0)):
        out = np.zeros(65536, np.int8)
        emul.lib().emul_feature_qlut(ctypes.c_float(scale), int(zp), out.ctypes.data_as(ctypes.c_void_p))
        assert np.array_equal(out, R.quantize_input(x, np.float32(scale), zp)), (scale, zp)


def test_closed_form_requantisation_equals_tflite_reference():
    """The kernels' MultiplyByQuantizedMultiplier (arithmetic-shift closed form) == the literal SRDHM + RoundingDivideByPOT."""
    from oracle import mixednet_ref as R
    L = emul.lib()
    L.emul_mbqm.restype = __import__("ctypes").c_int32
    rng = np.random.default_rng(5)
    xs = np.concatenate([rng.integers(-(1 << 31), 1 << 31, 3000), rng.integers(-70000, 70000, 3000),
                         np.array([0, 1, -1, (1 << 31) - 1, -(1 << 31), 1 << 30, -(1 << 30), 3 << 29, -(3 << 29)])]).astype(np.int64)
    cases = [(R.quantize_multiplier(m)) for m in (0.75, 0.5, 0.4999999, 0.0123, 0.00071, 0.999999, 1.0, 1.7, 3.2e-6)] + [(1 << 30, 0), ((1 << 31) - 1, 0), (1 << 30, -31), (0, 0)]
    for mult, shift in cases:
        if shift > 0:
            use = xs[np.abs(xs) < (1 << (30 - shift))]       # the reference's x * 2^left is int32 arithmetic; stay clear of overflow
        else:
            use = xs
        want = R.mbqm(use, mult, shift)
        got = np.array([L.emul_mbqm(int(x), int(mult), int(shift)) for x in use], np.int64)
        assert np.array_equal(got, np.asarray(want, np.int64)), (mult, shift)


def test_live_step_kernel_phases_match_oracle_and_interleave_with_clip():
    """Stream-parallel live-step kernel (one model step per call for many streams) == the oracle, for every pending-row
    phase (0, 1, 2), for a ragged last group (70 streams = 32 + 32 + 6), and it shares its state with the clip kernel."""
    t = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
    S = 70
    audio = np.stack([synth_audio(9600, 900 + i) for i in range(S)])
    feats, want = oracle.run_pipeline(MF.write_container(t), audio)            # 58 rows -> 19 probabilities
    for n_first, version, order in ((3, 2, 0), (4, 2, 1), (5, 2, 0), (4, 1, 0), (3, 3, 1), (4, 3, 0), (5, 3, 1)):   # first call leaves 0 / 1 / 2 rows pending
        nn = emul.NnF32Live(t, S, version=version, order=order)
        got = [nn.infer(feats[:, :n_first])]                                   # clip-kernel phases: 1 step (+ pending)
        pos = n_first
        while pos + 3 <= feats.shape[1]:
            got.append(nn.step(feats[:, pos:pos + 3])[:, None])                # live-step phases
            pos += 3
        got = np.concatenate(got, 1)
        assert np.abs(got - want[:, :got.shape[1]]).max() <= 1e-5, n_first
        # live calls keep the rings rotated; rotated back they are the clip kernel's state after the same rows
        assert nn.heads.any()
        ref = emul.NnF32(t, S)
        ref.infer(feats[:, :pos])
        nn.canonicalise()
        assert not nn.heads.any() and np.abs(nn.state - ref.state).max() <= 1e-5 and np.array_equal(nn.pend, ref.pend)
        # hand the state back to the clip kernel for the remaining rows: still the same chain
        rest = nn.infer(feats[:, pos:])
        tail = want[:, got.shape[1]:got.shape[1] + rest.shape[1]]
        assert rest.shape == tail.shape and (rest.size == 0 or np.abs(rest - tail).max() <= 1e-5)
    # the warp-specialised kernels perform the r01 kernel's arithmetic in the same order: bit-identical, state included -- also
    # with rows pending (a clip call of 4 rows first) and with float32 feature rows
    for first, dtype in ((0, np.float32), (4, np.float32), (5, np.uint16)):
        rows_all = feats if dtype == np.float32 else np.round(feats / np.float32(0.0390625)).astype(np.uint16)
        a, b, c = (emul.NnF32Live(t, S, version=v) for v in (1, 2, 3))
        if first:
            for e in (a, b, c):
                e.infer(feats[:, :first])
        for pos in range(first, first + 30, 3):
            pa = a.step(rows_all[:, pos:pos + 3])
            assert np.array_equal(pa, b.step(rows_all[:, pos:pos + 3])) and np.array_equal(pa, c.step(rows_all[:, pos:pos + 3]))
        assert np.array_equal(a.state, b.state) and np.array_equal(a.pend, b.pend)
        assert np.array_equal(a.state, c.state) and np.array_equal(a.pend, c.pend)
    # group-size edge cases: a single stream, one stream more than a full group
    for S2 in (1, 33):
        a, c = emul.NnF32Live(t, S2, version=1), emul.NnF32Live(t, S2, version=3, order=1)
        for e in (a, c):
            e.infer(feats[:S2, :4])
        for pos in range(4, 4 + 24, 3):
            assert np.array_equal(a.step(feats[:S2, pos:pos + 3]), c.step(feats[:S2, pos:pos + 3])), (S2, pos)
        assert np.array_equal(a.state, c.state) and np.array_equal(a.pend, c.pend)


def test_int8_live_step_kernel_phases_are_bit_exact():
    """int8 live-step kernel (IMMA, rotated int8 rings) == the integer oracle bit for bit: every pending-row phase, a
    ragged last group (70 streams), all three row dtypes, and a hand-over of the state to and from the clip kernel."""
    q = MF.load(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"))
    S = 70
    audio = np.concatenate([np.stack([synth_audio(9600, 950 + i) for i in range(S - 4)]), edge_case_audio(9600)[:4]])
    feats, want = oracle.run_pipeline(MF.write_container(q), audio)            # uint16 [70, 58, 40] -> 19 probabilities
    assert feats.dtype == np.uint16
    from oracle import mixednet_ref as R
    as_f32 = feats.astype(np.float32) * np.float32(0.0390625)
    as_i8 = R.quantize_input(as_f32, q["q/scales"][0], q["q/zps"][0])
    for rows, n_first in ((feats, 3), (feats, 4), (feats, 5), (as_f32, 4), (as_i8, 5)):
        nn = emul.NnI8Live(q, S)
        got = [nn.infer(rows[:, :n_first])]                                    # clip-kernel phases first (leaves 0 / 1 / 2 rows pending)
        pos = n_first
        while pos + 3 <= rows.shape[1]:
            got.append(nn.step(rows[:, pos:pos + 3])[:, None])                 # live-step phases
            pos += 3
        got = np.concatenate(got, 1)
        assert np.array_equal(got, want[:, :got.shape[1]]), (rows.dtype, n_first)
        assert nn.heads.any()
        ref = emul.NnI8(q, S)
        ref.infer(rows[:, :pos])
        nn.canonicalise()
        assert np.array_equal(nn.state, ref.state) and np.array_equal(nn.pend, ref.pend)
        rest = nn.infer(rows[:, pos:])
        assert np.array_equal(rest, want[:, got.shape[1]:got.shape[1] + rest.shape[1]])


def test_frontend_phases_bit_exact_property_based():
    """Hypothesis drives the amplitude structure instead of a fixed list: piecewise segments of silence, DC, full-scale
    clipping, alternating extremes, tones and noise at random levels, cut at arbitrary sample positions (so window
    boundaries fall anywhere), fed in two calls of arbitrary split.  Features must equal the oracle's bit for bit."""
    from hypothesis import given, settings, strategies as st

    seg = st.tuples(st.sampled_from(["zero", "dc", "clip", "alt", "tone", "noise", "impulse"]), st.integers(1, 900),
                    st.integers(0, 32767), st.integers(0, 2 ** 31 - 1))

    @settings(max_examples=40, deadline=None, derandomize=True)
    @given(st.lists(seg, min_size=1, max_size=8), st.integers(0, 4000))
    def run(segments, split):
        parts = []
        for kind, n, amp, seed in segments:
            r = np.random.default_rng(seed)
            t = np.arange(n)
            if kind == "zero":
                x = np.zeros(n)
            elif kind == "dc":
                x = np.full(n, amp if seed & 1 else -amp)
            elif kind == "clip":
                x = r.choice([-32768, 32767], n)
            elif kind == "alt":
                x = np.where(t % 2 == 0, amp, -amp - 1)
            elif kind == "tone":
                x = amp * np.sin(2 * np.pi * (50 + seed % 7900) / 16000.0 * t + seed % 7)
            elif kind == "noise":
                x = r.normal(0, amp / 3 + 1, n)
            else:
                x = np.zeros(n); x[seed % n] = amp if seed & 2 else -32768
            parts.append(x)
        audio = np.clip(np.round(np.concatenate(parts)), -32768, 32767).astype(np.int16)
        if audio.size < 480:
            audio = np.concatenate([audio, np.zeros(480 - audio.size, np.int16)])
        audio = audio[None]
        want, _ = oracle.run_pipeline(None, audio, want_probs=False)
        fe = emul.Frontend(1)
        cut = min(split, audio.shape[1])
        got = [fe.features(audio[:, :cut]), fe.features(audio[:, cut:])] if 0 < cut < audio.shape[1] else [fe.features(audio)]
        got = np.concatenate(got, 1)
        assert got.shape == want.shape and np.array_equal(got, want)

    run()
