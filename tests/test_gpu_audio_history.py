"""The audio history on the GPU (run with -m gpu on an H100).

Every read is compared bit for bit with the rule of include/mww.h applied to the input: a stream's history is zeros followed
by every 16 kHz sample its frontend consumed since it was last zeroed -- int16 as given, float32 as converted, G.711 as
decoded, other rates as tests/resample_oracle.py resamples the stream's whole input -- and a read returns the last n.  Beside
that: the carry identity (the last frontend_buffered history samples are the window carry), the resets that zero exactly the
rows the rule names, reads by a detector's fired_ids, bit-identity of everything else with a twin engine that keeps no
history, the launch count of a handle whose history is off, and refusals that leave the history unchanged."""

import ctypes
import os

import numpy as np
import pytest

import resample_oracle as ref
from conftest import GOLDEN
from microwakeword_b200 import _lib
from microwakeword_b200.detection import StreamDetector
from microwakeword_b200.engine import INPUT_RATES, MultiModelEngine, StreamEngine, inputs_for_rates, rate_inputs
from test_g711 import alaw_ref, ulaw_ref
from test_resample import taps

pytestmark = pytest.mark.gpu

P = 1021
F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
I8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")


def _blob(path):
    with open(path, "rb") as f:
        return f.read()


class Runs:
    """the rule: per stream, the 16 kHz samples appended since the last zeroing"""

    def __init__(self, S):
        self.r = [np.zeros(0, np.int16) for _ in range(S)]

    def add(self, samples, ids=None):
        for j, s in enumerate(range(len(self.r)) if ids is None else ids):
            self.r[s] = np.concatenate([self.r[s], np.asarray(samples[j], np.int16)])

    def zero(self, ids=None):
        for s in (range(len(self.r)) if ids is None else ids):
            self.r[s] = np.zeros(0, np.int16)

    def read(self, ids, n):
        out = np.zeros((len(ids), n), np.int16)
        for j, s in enumerate(ids):
            if 0 <= s < len(self.r) and n:
                t = self.r[s][-n:]
                out[j, n - t.size:] = t
        return out


def check(eng, runs, ids, n):
    got = eng.audio_history(list(ids), n).cpu().numpy()
    want = runs.read(list(ids), n)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]


def check_carry(eng, ids):
    d = eng.state_dict()
    fb = d["frontend_buffered"]
    if 0 < fb <= eng.audio_history_capacity:
        got = eng.audio_history(list(ids), fb).cpu().numpy()
        assert np.array_equal(got, d["carry"][list(ids), :fb])


def f32_to_int16(x):
    y = np.clip(np.asarray(x, np.float32) * np.float32(32768), -32768, 32767)
    return np.where(np.isnan(y), 0, y).astype(np.int16)


# ---- int16 at 65 536 streams: live calls, a clip longer than the ring, buffered samples, device-id reads, a twin ------------
def test_int16_at_65536_streams(torch_cuda):
    torch = torch_cuda
    S, C = 65536, 32000
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    base = torch.randint(-32768, 32768, (P, 100000), dtype=torch.int16, device="cuda", generator=g)
    idx = torch.arange(S, device="cuda") % P
    eng, twin = StreamEngine(F32, n_streams=S), StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    assert eng.audio_history_capacity == C and eng.audio_samples_seen == 0
    rng = np.random.default_rng(0)
    ids = np.concatenate([rng.choice(S, 300, replace=False), [0, S - 1, 5, 5]]).astype(np.int32)
    t = 0

    def call(n, step):
        nonlocal t
        audio = base[idx, t:t + n]
        a = eng.step(audio) if step else eng.predict_clip(audio)
        b = twin.step(audio) if step else twin.predict_clip(audio)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        t += n

    base_h = base.cpu().numpy()
    runs = lambda: [base_h[s % P, :t] for s in ids]                   # noqa: E731

    for i in range(100):                                              # 2 s of live calls: the ring wraps at 32 000
        call(480, True)
        if i in (10, 70):
            assert np.array_equal(eng.audio_history(ids, C).cpu().numpy(), Runs_read(runs(), C))
    call(48000, False)                                                # the fused clip kernel; longer than the ring
    call(100, False)                                                  # leaves samples buffered
    call(37, False)                                                   # scalar append
    assert eng.audio_samples_seen == t == 96137
    want = Runs_read(runs(), C)
    assert np.array_equal(eng.audio_history(ids, C).cpu().numpy(), want)
    assert np.array_equal(eng.audio_history(ids, 1).cpu().numpy(), want[:, -1:])
    assert eng.audio_history(ids, 0).shape == (len(ids), 0)
    d_ids = torch.from_numpy(np.concatenate([ids, [-1, S, -7]]).astype(np.int32)).cuda()
    got = eng.audio_history(d_ids, 24000).cpu().numpy()
    assert np.array_equal(got[:len(ids)], want[:, -24000:]) and not got[len(ids):].any()
    out = torch.full((len(ids), 24003), 7, dtype=torch.int16, device="cuda")
    eng.audio_history(ids, 24000, out=out[:, 3:])                     # rows misaligned: the scalar read
    assert np.array_equal(out[:, 3:].cpu().numpy(), want[:, -24000:]) and (out[:, :3] == 7).all()
    a, b = eng.state_dict(), twin.state_dict()
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    fb = a["frontend_buffered"]
    assert np.array_equal(eng.audio_history(ids, fb).cpu().numpy(), a["carry"][ids, :fb])
    eng.close(); twin.close()
    del base
    torch.cuda.empty_cache()


def Runs_read(rows, n):
    r = Runs(len(rows))
    r.r = [np.asarray(x, np.int16) for x in rows]
    return r.read(list(range(len(rows))), n)


# ---- every sample type, the vector and scalar loads, the K1 + K2 path and the run-time hop ----------------------------------
def test_sample_types_and_load_forms(torch_cuda):
    torch = torch_cuda
    S, C = 256, 4096
    rng = np.random.default_rng(1)
    eng = StreamEngine(None, n_streams=S)
    eng.set_audio_history(C)
    runs = Runs(S)
    for kind in ("int16", "float32", "ulaw", "alaw", "int16", "ulaw", "float32", "alaw"):
        for n, off, extra in ((480, 0, 0), (160, 0, 0), (1000, 1, 0), (203, 0, 5), (4800, 0, 8), (7, 3, 1), (5000, 0, 0)):
            w = off + n + extra
            if kind == "int16":
                host = rng.integers(-32768, 32768, (S, w), dtype=np.int64).astype(np.int16)
                want, law = host, None
            elif kind == "float32":
                host = (rng.standard_normal((S, w)) * 0.5).astype(np.float32)
                host[0, :3] = (np.nan, 2.0, -2.0)
                want, law = f32_to_int16(host), None
            else:
                host = rng.integers(0, 256, (S, w), dtype=np.int64).astype(np.uint8)
                want, law = (ulaw_ref(host) if kind == "ulaw" else alaw_ref(host)), kind
            dev = torch.from_numpy(host).cuda()[:, off:off + n]       # offset: misaligned rows; extra: a pitch not a multiple of 8
            eng.features(dev, law=law)
            runs.add(want[:, off:off + n])
        check(eng, runs, range(0, S, 7), C)
        check(eng, runs, [3, 3, 200], 1)
    check_carry(eng, range(S))
    eng.reset()
    runs.zero()
    eng.set_window_step(320)                                          # the run-time-hop kernel
    for n in (960, 333, 4000):
        host = rng.integers(-32768, 32768, (S, n), dtype=np.int64).astype(np.int16)
        eng.features(torch.from_numpy(host).cuda())
        runs.add(host)
        check(eng, runs, range(S), C)
    check_carry(eng, range(S))
    eng.close()


# ---- resampled input: 8 and 48 kHz handles, per-stream rates over all seven ------------------------------------------------
@pytest.mark.parametrize("rate", [8000, 48000])
def test_one_input_rate(torch_cuda, rate):
    torch = torch_cuda
    S, C = 64, 8000
    rng = np.random.default_rng(rate)
    eng = StreamEngine(F32, n_streams=S, input_rate=rate)
    eng.set_audio_history(C)
    x = np.zeros((S, 0), np.int16)
    for n in (rate // 100 * 3, 1, 7777, rate * 3 // 2, 240, 3):
        a = rng.integers(-20000, 20000, (S, n), dtype=np.int64).astype(np.int16)
        eng.predict_clip(torch.from_numpy(a).cuda())
        x = np.concatenate([x, a], 1)
        y = ref.resample(x, taps(rate)[0], rate)
        assert eng.audio_samples_seen == y.shape[1]
        r = Runs(S); r.r = list(y)
        check(eng, r, range(S), C)
    check_carry(eng, range(S))
    # the staged path resamples tile by tile
    a = rng.integers(-20000, 20000, (S, rate), dtype=np.int64).astype(np.int16)
    eng.predict_clip_host(a)
    x = np.concatenate([x, a], 1)
    r = Runs(S); r.r = list(ref.resample(x, taps(rate)[0], rate))
    check(eng, r, range(S), C)
    eng.close()


def test_per_stream_rates(torch_cuda):
    torch = torch_cuda
    S, C = 70, 4000
    rng = np.random.default_rng(7)
    rates = np.array([INPUT_RATES[s % len(INPUT_RATES)] for s in range(S)], np.int32)
    eng = StreamEngine(F32, n_streams=S, stream_rates=rates)
    eng.set_audio_history(C)
    xs = [np.zeros(0, np.int16) for _ in range(S)]
    t = 0
    for n16 in (480, 2, 6400, 480, 960, 10000):
        D = inputs_for_rates(rates, t, n16)
        a = rng.integers(-20000, 20000, (S, int(D.max())), dtype=np.int64).astype(np.int16)
        eng.predict_clip(torch.from_numpy(a).cuda(), samples16=n16)
        for s in range(S):
            xs[s] = np.concatenate([xs[s], a[s, :D[s]]])
        t += n16
    assert eng.audio_samples_seen == t
    r = Runs(S)
    for s in range(S):
        assert xs[s].size == rate_inputs(t, int(rates[s]))
        r.r[s] = xs[s] if rates[s] == 16000 else ref.resample(xs[s], taps(int(rates[s]))[0], int(rates[s]))[:t]
    check(eng, r, range(S), C)
    check_carry(eng, range(S))
    # set_stream_rates leaves every row alone
    eng.set_stream_rates([0, 1], [48000, 8000])
    check(eng, r, range(S), C)
    eng.close()


# ---- host and remote calls, in place and staged over several tiles; multi-model handles with stream sets ---------------------
def test_host_and_remote_calls(torch_cuda):
    torch = torch_cuda
    S, C = 8192, 16000
    rng = np.random.default_rng(11)
    eng, twin = StreamEngine(F32, n_streams=S), StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    runs = Runs(S)
    ids = list(rng.choice(S, 200, replace=False)) + [0, S - 1]
    pinned = eng.host_buffer((S, 4000))
    for form in ("pageable", "pinned", "remote", "staged", "pageable", "staged"):
        n = {"pageable": 4000 - 3, "pinned": 4000, "remote": 480, "staged": 2400}[form]
        a = rng.integers(-32768, 32768, (S, n), dtype=np.int64).astype(np.int16)
        if form in ("pageable", "pinned"):
            src = a if form == "pageable" else pinned[:, :n]
            src[...] = a
            p, q = eng.predict_clip_host(src), twin.predict_clip_host(src)
            assert np.array_equal(p.view(np.int32), q.view(np.int32))
        else:
            dev = torch.from_numpy(a).cuda()
            tiles = 4 if form == "staged" else 0
            p = eng.predict_clip_remote(dev.data_ptr(), n, tiles=tiles)
            q = twin.predict_clip_remote(dev.data_ptr(), n, tiles=tiles)
            assert torch.equal(p.view(torch.int32), q.view(torch.int32))
        runs.add(a)
        check(eng, runs, ids, C)
    check_carry(eng, ids)
    a, b = eng.state_dict(), twin.state_dict()
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    eng.close(); twin.close()


def test_multi_model_with_stream_sets(torch_cuda):
    torch = torch_cuda
    S, C = 512, 8000
    rng = np.random.default_rng(13)
    sets = [np.arange(0, S, 3, dtype=np.int32), np.arange(100, 300, dtype=np.int32)]
    eng = MultiModelEngine([F32, I8], n_streams=S, streams=sets)
    twin = MultiModelEngine([F32, I8], n_streams=S, streams=sets)
    eng.set_audio_history(C)
    runs = Runs(S)
    for n in (480, 480, 3000, 77, 480):
        a = rng.integers(-32768, 32768, (S, n), dtype=np.int64).astype(np.int16)
        dev = torch.from_numpy(a).cuda()
        for p, q in zip(eng.predict_clip(dev), twin.predict_clip(dev)):
            assert torch.equal(p.view(torch.int32), q.view(torch.int32))
        runs.add(a)
    check(eng, runs, range(S), C)                                     # every stream, member or not
    eng.close(); twin.close()


# ---- zeroing ---------------------------------------------------------------------------------------------------------------
def test_resets_zero_exactly_the_named_rows(torch_cuda):
    torch = torch_cuda
    S, C = 300, 2000
    rng = np.random.default_rng(17)
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    runs = Runs(S)

    def feed(n=700):
        a = rng.integers(-32768, 32768, (S, n), dtype=np.int64).astype(np.int16)
        eng.predict_clip(torch.from_numpy(a).cuda())
        runs.add(a)

    feed()
    eng.reset([3, 17, 250])
    runs.zero([3, 17, 250])
    check(eng, runs, range(S), C)
    feed()
    eng.reset(torch.tensor([5, -1, 299, 5], dtype=torch.int32, device="cuda"))
    runs.zero([5, 299])
    check(eng, runs, range(S), C)
    feed()
    seen = eng.audio_samples_seen
    eng.reset_frontend()
    runs.zero()
    check(eng, runs, range(S), C)
    feed()
    eng.reset()
    runs.zero()
    check(eng, runs, range(S), C)
    assert eng.audio_samples_seen == seen + 700                       # resets do not clear the counter
    feed(480)
    feed(480)
    # import zeroes the rows it writes; export leaves the source alone
    src = StreamEngine(F32, n_streams=S)
    src.set_audio_history(C)
    for _ in range(2):
        src.predict_clip(torch.zeros((S, 480), dtype=torch.int16, device="cuda"))
    rec = src.export_streams([1, 2, 40])
    eng.import_streams([10, 11, 12], rec)
    runs.zero([10, 11, 12])
    check(eng, runs, range(S), C)
    # set_state leaves every row alone
    d = eng.state_dict()
    eng.load_state_dict(d)
    check(eng, runs, range(S), C)
    # set_audio_history zeroes every stream and restarts the counter
    eng.set_audio_history(C // 2)
    runs.zero()
    assert eng.audio_samples_seen == 0
    check(eng, runs, range(S), C // 2)
    feed(480)
    check(eng, runs, range(S), C // 2)
    check_carry(eng, range(S))
    eng.close(); src.close()


def test_read_by_detector_fired_ids(torch_cuda):
    torch = torch_cuda
    S, C = 1024, 8000
    rng = np.random.default_rng(19)
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    det = StreamDetector(S, cutoff=-1.0, window=1, cooldown_slices=2, capacity=3 * S)    # each row fires once, on its 2nd step
    runs = Runs(S)
    for _ in range(3):
        a = rng.integers(-32768, 32768, (S, 480), dtype=np.int64).astype(np.int16)
        det.update(eng.step(torch.from_numpy(a).cuda()))
        runs.add(a)
    clips = eng.audio_history(det.fired_ids, 1440)                    # before the drain
    fired = det.fired_ids.cpu().numpy()
    assert (fired >= 0).sum() == S and (fired < 0).any()
    want = runs.read(list(fired), 1440)
    assert np.array_equal(clips.cpu().numpy(), want)
    assert not want[fired < 0].any()
    eng.reset(det.fired_ids)
    det.drain()
    runs.zero()
    check(eng, runs, range(S), C)
    eng.close()


# ---- nothing else changes --------------------------------------------------------------------------------------------------
def test_twin_bit_identity_and_launch_counts(torch_cuda):
    torch = torch_cuda
    S = 512
    rng = np.random.default_rng(23)
    on, off, back = (StreamEngine(I8, n_streams=S) for _ in range(3))
    never = StreamEngine(I8, n_streams=S)
    on.set_audio_history(800)
    back.set_audio_history(64)
    back.set_audio_history(0)
    assert back.audio_history_capacity == 0
    for n in (480, 480, 3000, 50, 480):
        a = torch.from_numpy(rng.integers(-32768, 32768, (S, n), dtype=np.int64).astype(np.int16)).cuda()
        outs = [e.predict_clip(a) for e in (on, off, back, never)]
        for o in outs[1:]:
            assert torch.equal(outs[0].view(torch.int32), o.view(torch.int32))
        f = [e.features(a[:, :100]) for e in (on, off, back, never)]
        for o in f[1:]:
            assert torch.equal(f[0], o)
    on.reset([1, 2]); off.reset([1, 2]); back.reset([1, 2]); never.reset([1, 2])
    ref_state = off.state_dict()
    for e in (on, back, never):
        d = e.state_dict()
        for k in ref_state:
            assert np.array_equal(np.asarray(d[k]), np.asarray(ref_state[k])), k
    assert back.launch_count == off.launch_count == never.launch_count
    assert on.launch_count > off.launch_count
    for e in (on, off, back, never):
        e.close()


def test_refusals_leave_the_history_unchanged(torch_cuda):
    torch = torch_cuda
    S, C = 64, 512
    rng = np.random.default_rng(29)
    eng = StreamEngine(None, n_streams=S)
    L, h = eng._L, eng._h
    st = eng._cu_stream()
    with pytest.raises(ValueError):
        eng.audio_history([0], 8)                                     # no history yet
    out0 = torch.zeros((1, 8), dtype=torch.int16, device="cuda")
    assert L.mww_read_audio_history(h, np.zeros(1, np.int32).ctypes.data, 1, 8, out0.data_ptr(), 8, st) == -1
    eng.set_audio_history(C)
    a = rng.integers(-32768, 32768, (S, 900), dtype=np.int64).astype(np.int16)
    eng.features(torch.from_numpy(a).cuda())
    runs = Runs(S)
    runs.add(a)
    before = eng.audio_history(range(S), C).clone()
    out = torch.zeros((4, C), dtype=torch.int16, device="cuda")
    ids = np.array([0, 1, 2, S], np.int32)
    d_ids = torch.zeros(4, dtype=torch.int32, device="cuda")
    for rc in (L.mww_set_audio_history(h, 12, st), L.mww_set_audio_history(h, -8, st), L.mww_set_audio_history(h, (1 << 22) + 8, st),
               L.mww_read_audio_history(h, ids.ctypes.data, 4, 8, out.data_ptr(), C, st),          # id out of range
               L.mww_read_audio_history(h, ids.ctypes.data, -1, 8, out.data_ptr(), C, st),
               L.mww_read_audio_history_device_ids(h, d_ids.data_ptr(), 4, C + 8, out.data_ptr(), C + 8, st),
               L.mww_read_audio_history_device_ids(h, d_ids.data_ptr(), 4, 16, out.data_ptr(), 8, st),
               L.mww_read_audio_history_device_ids(h, None, 4, 16, out.data_ptr(), 16, st),
               L.mww_read_audio_history_device_ids(h, d_ids.data_ptr(), 4, 16, None, 16, st)):
        assert rc == -1
    assert not out.any()
    big = StreamEngine(None, n_streams=65536)
    big.set_audio_history(8)
    with pytest.raises(_lib.MwwError) as e:
        big.set_audio_history(1 << 22)                                # 512 GB
    assert e.value.code == -4 and big.audio_history_capacity == 8
    big.close()
    assert eng.audio_history_capacity == C and eng.audio_samples_seen == 900
    assert torch.equal(eng.audio_history(range(S), C), before)
    check(eng, runs, range(S), C)
    eng.close()
