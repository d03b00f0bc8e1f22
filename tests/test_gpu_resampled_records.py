"""Moving resampled streams between handles (mww_export_resampled_streams / mww_import_resampled_streams), run with -m gpu on
an H100.  The reference is the source left in place: a moved stream's probabilities, state and resampler history must equal
the source stream's, bit for bit, after further calls of random lengths.  The models are int8 (exact at any ring rotation).
Covered: every single-rate handle with int16, float32 and (8 kHz) G.711 audio; a 65 536-stream handle with all seven rates
grown into 98 304 streams; moves across modes; the phase and rate refusals at 22.05 kHz, which leave both handles unchanged;
a whole serving move on an 8 kHz mu-law handle while commands are spoken; a multi-model handle with stream subsets and
mixed rates; and the launch counts."""

import os

import numpy as np
import pytest

from conftest import GOLDEN
from microwakeword_b200 import _lib

pytestmark = pytest.mark.gpu

I8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
RATES = (8000, 16000, 22050, 24000, 32000, 44100, 48000)
H = {8000: 52, 16000: 0, 22050: 111, 24000: 122, 32000: 163, 44100: 222, 48000: 243}
LAW = {"ulaw": "ulaw", "alaw": "alaw"}


def _gen(torch, kind, S, n, g):
    if kind in LAW:
        return torch.randint(0, 256, (S, n), dtype=torch.uint8, device="cuda", generator=g)
    x = torch.randint(-9000, 9000, (S, n), dtype=torch.int16, device="cuda", generator=g)
    return x if kind == "int16" else (x.to(torch.float32) / 32768.0)


def _call(eng, x, kind, n16=None):
    return eng.predict_clip(x, samples16=n16, law=LAW.get(kind))


def _bits(p):
    return p.cpu().numpy().view(np.int32)


def _rows(eng, ids):
    """the per-stream state of streams ids: frontend, model, and each stream's own H resampler samples"""
    d = eng.state_dict()
    out = {k: d[k][ids] for k in ("carry", "estimate", "nn", "pending") if k in d}
    rates = eng.stream_rates[ids]
    hist = d.get("resampler_history")
    out["resampler"] = [hist[s, :H[int(r)]] if hist is not None else np.zeros(0, np.int16) for s, r in zip(ids, rates)]
    if hist is not None and eng.per_stream_rates:          # the rest of a per-stream row is zero
        for s, r in zip(ids, rates):
            assert not hist[s, H[int(r)]:].any(), (s, r)
    return out


def _assert_rows_equal(a, b, what):
    for k in a:
        if k == "resampler":
            assert all(np.array_equal(x, y) for x, y in zip(a[k], b[k])), (what, k)
        else:
            assert np.array_equal(a[k], b[k]), (what, k)


class Pair:
    """a source and a destination handle fed in lockstep: stream dst[i] of the destination hears what src[i] of the source
    hears; every other destination stream hears its own audio"""

    def __init__(self, torch, A, B, seed):
        self.torch, self.A, self.B = torch, A, B
        self.g = torch.Generator(device="cuda").manual_seed(seed)
        self.src = self.dst = None

    def width(self, eng, n):
        return int(eng.inputs_for(n).max()) if eng.per_stream_rates else n

    def call(self, n, kind="int16", nb=None):
        """n: input samples of a single-rate handle, or n16 of a per-stream one (nb: the destination's, default n)"""
        t = self.torch
        nb = n if nb is None else nb
        wa, wb = self.width(self.A, n), self.width(self.B, nb)
        a, b = _gen(t, kind, self.A.n_streams, wa, self.g), _gen(t, kind, self.B.n_streams, wb, self.g)
        if self.src is not None:
            w = min(wa, wb)
            b[t.from_numpy(self.dst).long().cuda(), :w] = a[t.from_numpy(self.src).long().cuda(), :w]
        n16a = n if self.A.per_stream_rates else None
        n16b = nb if self.B.per_stream_rates else None
        return _call(self.A, a, kind, n16a), _call(self.B, b, kind, n16b)

    def move(self, src, dst, **kw):
        self.src, self.dst = np.asarray(src, np.int32), np.asarray(dst, np.int32)
        recs = self.A.export_streams(self.src, resampler=True, **kw)
        if self.B.per_stream_rates:
            self.B.set_stream_rates(self.dst, recs.rates)
        self.B.import_streams(self.dst, recs)
        return recs

    def check(self, pa, pb, what):
        assert pa.shape[1] == pb.shape[1], what
        assert np.array_equal(_bits(pb)[self.dst], _bits(pa)[self.src]), what

    def check_state(self, what):
        _assert_rows_equal(_rows(self.A, self.src), _rows(self.B, self.dst), what)


# ---- 1. every single-rate handle ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", RATES)
def test_every_single_rate_handle(torch_cuda, rate):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    SA, SB = 700, 1100
    kinds = ["int16", "float32"] + (["ulaw", "alaw"] if rate == 8000 else [])
    rng = np.random.default_rng(rate)
    A, B = StreamEngine(I8, SA, input_rate=rate), StreamEngine(I8, SB, input_rate=rate)
    p = Pair(torch, A, B, rate)
    for n in (rate * 5 // 16 + 7, 3 * rate // 100, 3 * rate // 100 + 1):       # ~0.3 s: pending rows and buffered samples
        p.call(n)
    assert A.frontend_buffered > 0
    src, dst = rng.permutation(SA)[:300], rng.permutation(SB)[:300]
    recs = p.move(src, dst)
    assert recs.resampler.rate == rate and np.all(recs.rates == rate)
    assert recs.data.shape[1] == recs.resampler.record_bytes == recs.layout.record_bytes + 496
    steps = 0
    for i in range(8):
        kind = kinds[i % len(kinds)]
        pa, pb = p.call(int(rng.integers(1, rate // 5)), kind)
        p.check(pa, pb, (rate, i, kind))
        steps += pa.shape[1]
    assert steps > 0
    p.check_state(rate)
    assert A._rate()[1] == B._rate()[1]


# ---- 2. a per-stream handle at full size -------------------------------------------------------------------------------------
def test_per_stream_handle_grown_at_full_size(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S, Sd = 65536, 98304
    rng = np.random.default_rng(2)
    rates_a = np.asarray(RATES, np.int32)[rng.integers(0, 7, S)]
    rates_a[:7] = RATES
    A = StreamEngine(I8, S, stream_rates=rates_a)
    B = StreamEngine(I8, Sd, stream_rates=np.asarray(RATES, np.int32)[rng.integers(0, 7, Sd)])
    p = Pair(torch, A, B, 20)
    for n in (4802, 480, 480):
        p.call(n)
    dst = rng.permutation(Sd)[:S]
    recs = p.move(np.arange(S), dst)
    assert recs.resampler.rate == _lib.MWW_RATE_PER_STREAM and np.array_equal(recs.rates, rates_a)
    assert np.array_equal(B.stream_rates[dst], rates_a)
    for i, n in enumerate((480, 962, 480)):
        pa, pb = p.call(n)
        p.check(pa, pb, i)
    p.check_state("full size")


# ---- 3. moves across modes ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("law", ["ulaw", "alaw"])
def test_g711_8k_into_per_stream_slots_and_back(torch_cuda, law):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    rng = np.random.default_rng(8)
    S, Sd = 600, 900
    A = StreamEngine(I8, S, input_rate=8000)
    B = StreamEngine(I8, Sd, stream_rates=np.asarray(RATES, np.int32)[rng.integers(0, 7, Sd)])
    p = Pair(torch, A, B, 81)
    for n in (2401, 240, 240):                       # n 8 kHz samples are 2 n 16 kHz samples
        p.call(n, law, nb=2 * n)
    src, dst = rng.permutation(S)[:250], rng.permutation(Sd)[:250]
    p.move(src, dst)
    assert np.all(B.stream_rates[dst] == 8000)
    for i in range(4):
        n = int(rng.integers(1, 900))
        pa, pb = p.call(n, law, nb=2 * n)
        p.check(pa, pb, ("in", i))
    p.check_state("into per-stream")
    # and back: into a single-rate 8 kHz handle whose counters match
    C = StreamEngine(I8, S + 50, input_rate=8000)
    back = Pair(torch, B, C, 82)
    t = B._rate()[1]
    C.predict_clip(_gen(torch, law, C.n_streams, t // 2, back.g), law=law)     # t 16 kHz samples: the same frontend counters
    back.move(dst, rng.permutation(S + 50)[:250])
    for i in range(4):
        n = 2 * int(rng.integers(1, 450))
        pb, pc = back.call(n, law, nb=n // 2)
        back.check(pb, pc, ("back", i))
    back.check_state("back to single rate")


def test_plain_16k_into_per_stream_slots_at_16000(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    rng = np.random.default_rng(16)
    A = StreamEngine(I8, 500)
    B = StreamEngine(I8, 800, stream_rates=np.asarray(RATES, np.int32)[rng.integers(0, 7, 800)])
    p = Pair(torch, A, B, 160)
    for n in (4802, 480):
        p.call(n)
    recs = p.move(rng.permutation(500)[:200], rng.permutation(800)[:200])
    assert recs.resampler.rate == 16000 and not recs.data[:, recs.resampler.resampler_off:].any()
    for i in range(3):
        n = 2 * int(rng.integers(1, 1500))
        pa, pb = p.call(n)
        p.check(pa, pb, i)
    p.check_state("16 kHz into per-stream")


# ---- 4. refusals at 22.05 kHz -----------------------------------------------------------------------------------------------
def _snapshot(eng):
    torch = __import__("torch")
    torch.cuda.synchronize()
    d = eng.state_dict()
    return {k: (np.asarray(v).copy() if isinstance(v, np.ndarray) else v) for k, v in d.items()}, eng.launch_count


def _same(a, b):
    assert a[1] == b[1]
    assert a[0].keys() == b[0].keys()
    for k in a[0]:
        assert np.array_equal(np.asarray(a[0][k]), np.asarray(b[0][k])), k


def test_22050_phase_and_rate_refusals(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    rng = np.random.default_rng(22)
    A, B2 = StreamEngine(I8, 400, input_rate=22050), StreamEngine(I8, 500, input_rate=22050)
    q = Pair(torch, A, B2, 221)
    for n in (661, 662, 661):                       # 30 ms calls: three on the source, two on the destination
        A.predict_clip(_gen(torch, "int16", 400, n, q.g))
    for n in (661, 662):
        B2.predict_clip(_gen(torch, "int16", 500, n, q.g))
    src, dst = rng.permutation(400)[:100].astype(np.int32), rng.permutation(500)[:100].astype(np.int32)
    assert A._rate()[1] % 441 == 220 and B2._rate()[1] % 441 == 0          # half a cycle apart
    recs = A.export_streams(src, resampler=True)
    before_a, before_b = _snapshot(A), _snapshot(B2)
    with pytest.raises(_lib.MwwError) as e:
        B2.import_streams(dst, recs)
    assert "phase" in str(e.value) and "22050 Hz" in str(e.value) and "= 220" in str(e.value) and "handle's 0" in str(e.value)
    _same(before_a, _snapshot(A))
    _same(before_b, _snapshot(B2))
    # a rate mismatch: the same records into a 24 kHz handle with matching frontend counters
    C = StreamEngine(I8, 500, input_rate=24000)
    for n in (720, 720, 720):
        C.predict_clip(_gen(torch, "int16", 500, n, q.g))
    before_c = _snapshot(C)
    with pytest.raises(_lib.MwwError) as e:
        C.import_streams(dst, recs)
    assert "24000" in str(e.value) and "rate" in str(e.value)
    _same(before_c, _snapshot(C))
    # one more call on the destination and the move is accepted, and exact
    q.B.predict_clip(_gen(torch, "int16", 500, 661, q.g))
    assert B2._rate()[1] % 441 == 220
    q.src, q.dst = src, dst
    B2.import_streams(dst, A.export_streams(src, resampler=True))
    for i in range(4):
        pa, pb = q.call(int(rng.integers(1, 3000)))
        q.check(pa, pb, i)
    q.check_state("22.05 kHz after one more call")


# ---- 5. a whole serving move on an 8 kHz mu-law handle while commands are spoken ----------------------------------------------
RULE = dict(vad_window=5, vad_cutoff=0.5, speech_steps=3, silence_steps=8, timeout_steps=100, max_steps=120, lookback_steps=12)


def _script(S, steps, rng):
    j = np.arange(steps)[None, :]
    period = rng.integers(3, 14, S)[:, None]
    phase = rng.integers(0, 40, S)[:, None]
    return np.where(((j + phase) // period) % 2 == 0, 0.9, 0.05).astype(np.float32)


def _sorted(ev):
    return ev[np.lexsort((ev["stream"], ev["end_sample"]))]


def test_serving_move_on_8k_ulaw_while_commands_are_spoken(torch_cuda):
    from microwakeword_b200.detection import StreamDetector
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S, Sd, C = 4096, 6000, 32000
    PRE, POST, MAX, CAP = 1600, 3200, 32000, 4096
    BEFORE, AFTER, DST_BEFORE = 120, 90, 40
    rng = np.random.default_rng(5)
    P = _script(S, BEFORE + AFTER, rng)
    g = torch.Generator(device="cuda").manual_seed(55)
    src = StreamEngine(I8, S, input_rate=8000)
    src.set_audio_history(C)
    ep = Endpointer(src, capacity=CAP, **RULE)
    det = StreamDetector(S, cutoff=0.9)
    arms = {59: rng.choice(S, 600, replace=False), 99: rng.choice(S, 600, replace=False), 114: rng.choice(S, 600, replace=False),
            139: rng.choice(S, 600, replace=False), 169: rng.choice(S, 600, replace=False)}
    used = 0
    for c in range(BEFORE):
        pr = src.step(torch.randint(0, 256, (S, 240), dtype=torch.uint8, device="cuda", generator=g), law="ulaw")
        det.update(pr)
        n = pr.shape[1]
        ep.update(torch.from_numpy(P[:, used:used + n]).cuda())
        used += n
        if c % 5 == 4:
            ep.drain()
            det.drain()
        if c in arms:
            ep.arm(arms[c])
    assert (ep.state_dict()["armed"] >= 0).sum() > 0
    dst = StreamEngine(I8, Sd, stream_rates=np.asarray(RATES, np.int32)[rng.integers(0, 7, Sd)])
    dst.set_audio_history(C)
    dep = Endpointer(dst, capacity=CAP, **RULE)
    ddet = StreamDetector(Sd, cutoff=0.9)
    for c in range(DST_BEFORE):
        w = int(dst.inputs_for(480).max())
        pr = dst.step(torch.randint(0, 256, (Sd, w), dtype=torch.uint8, device="cuda", generator=g), law="ulaw")
        ddet.update(pr)
        dep.update(torch.rand((Sd, pr.shape[1]), device="cuda"))
    dep.drain()
    ddet.drain()
    # the move, in the README's order: rates, stream records with the resampler and the history, detector rows, endpointer rows
    to = rng.permutation(Sd)[:S].astype(np.int32)
    shift = dst.audio_samples_seen - src.audio_samples_seen
    ids = np.arange(S, dtype=np.int32)
    dst.set_stream_rates(to, 8000)
    for b in range(0, S, 1024):
        recs = src.export_streams(ids[b:b + 1024], history=C, resampler=True)
        dst.import_streams(to[b:b + 1024], recs)
    ddet.import_rows(to, det.export_rows(ids))
    dep.import_streams(to, ep.export_streams(ids))
    to_t = torch.from_numpy(to).long().cuda()
    got_ev, want_ev = [], []
    for c in range(BEFORE, BEFORE + AFTER):
        a = torch.randint(0, 256, (S, 240), dtype=torch.uint8, device="cuda", generator=g)
        w = int(dst.inputs_for(480).max())
        b = torch.randint(0, 256, (Sd, w), dtype=torch.uint8, device="cuda", generator=g)
        b[to_t, :240] = a
        pr, prd = src.step(a, law="ulaw"), dst.step(b, law="ulaw")
        assert np.array_equal(_bits(prd)[to], _bits(pr)), c
        det.update(pr)
        ddet.update(prd)
        n = pr.shape[1]
        ps = torch.from_numpy(P[:, used:used + n]).cuda()
        used += n
        pd = torch.rand((Sd, n), device="cuda") * 0.4
        pd[to_t] = ps
        ep.update(ps)
        dep.update(pd)
        if c % 5 == 4:
            clips, lens = ep.commands(PRE, POST, MAX)
            dclips, dlens = dep.commands(PRE, POST, MAX)
            torch.cuda.synchronize()
            ev, n = ep._drain_slots()
            dev_, dn = dep._drain_slots()
            assert n == dn
            slot = {int(s): i for i, s in enumerate(dev_["stream"])}
            j = torch.tensor([slot[int(to[s])] for s in ev["stream"]], dtype=torch.long, device="cuda")
            if ev.size:
                assert torch.equal(lens[:ev.size], dlens[j]) and torch.equal(clips[:ev.size], dclips[j]), c
            m = ev.copy()
            m["stream"] = to[ev["stream"]]
            for k in ("start_sample", "end_sample", "speech_end_sample"):
                m[k] += shift
            want_ev.append(m)
            got_ev.append(dev_)
        if c in arms:
            ep.arm(arms[c])
            dep.arm(to[arms[c]])
    want, got = _sorted(np.concatenate(want_ev)), _sorted(np.concatenate(got_ev))
    assert want.size > 100 and np.array_equal(got, want)


# ---- 6. multi-model handles --------------------------------------------------------------------------------------------------
def test_multi_model_stream_subsets_and_mixed_rates(torch_cuda):
    from microwakeword_b200.engine import MultiModelEngine
    from test_gpu_multi_model import _blobs
    torch = torch_cuda
    blobs = [_blobs()[i] for i in (1, 4)]               # int8 okay_nabu, int8 run-time geometry of stride 17
    rng = np.random.default_rng(6)
    SA, SB = 900, 1300
    src, dst = rng.permutation(SA)[:400].astype(np.int32), rng.permutation(SB)[:400].astype(np.int32)
    sets_a = [None, np.arange(0, SA, 2, dtype=np.int32)]
    member = src % 2 == 0
    sets_b = [np.union1d(dst[member], np.arange(0, SB, 5)).astype(np.int32), None]
    keep = np.isin(dst, sets_b[0])                      # moved streams that are members of model 0 on both sides ...
    rates = lambda S: np.asarray(RATES, np.int32)[rng.integers(0, 7, S)]  # noqa: E731
    A = MultiModelEngine(blobs, SA, streams=sets_a, stream_rates=rates(SA))
    B = MultiModelEngine(blobs, SB, streams=sets_b, stream_rates=rates(SB))
    p = Pair(torch, A, B, 60)
    for n in (4802, 480, 480):
        p.call(n)
    p.move(src, dst)
    for n in (480, 2002, 480, 480):
        p.call(n)
    torch.cuda.synchronize()
    sa, sb = A.state_dict(), B.state_dict()
    for key in ("carry", "estimate"):
        assert np.array_equal(sb[key][dst], sa[key][src]), key
    hb, ha = sb["resampler_history"], sa["resampler_history"]
    assert np.array_equal(hb[dst], ha[src])
    for k, (ok_src, ok_dst) in enumerate(((src[keep], dst[keep]), (src[member], dst[member]))):
        ma, mb = sa["models"][k], sb["models"][k]
        ia = np.searchsorted(ma["streams"], ok_src)
        ib = np.searchsorted(mb["streams"], ok_dst)
        assert np.array_equal(ma["streams"][ia], ok_src) and np.array_equal(mb["streams"][ib], ok_dst)
        assert ok_src.size > 50
        for key in ("nn", "pending"):
            assert np.array_equal(mb[key][ib], ma[key][ia]), (k, key)


# ---- 7. launch counts --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 65536])
def test_launch_counts_are_the_old_pairs_plus_one(torch_cuda, n):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    S = 65536
    plain, r48 = StreamEngine(I8, S), StreamEngine(I8, S, input_rate=48000)
    plain.set_audio_history(480)
    r48.set_audio_history(480)
    plain.step(torch.zeros((S, 480), dtype=torch.int16, device="cuda"))
    r48.step(torch.zeros((S, 1440), dtype=torch.int16, device="cuda"))
    ids = np.random.default_rng(n).permutation(S)[:n]

    def counted(eng, fn):
        L0 = eng.launch_count
        out = fn()
        return eng.launch_count - L0, out

    old_exp, recs = counted(plain, lambda: plain.export_streams(ids))
    old_imp, _ = counted(plain, lambda: plain.import_streams(ids, recs))
    for eng in (plain, r48):
        exp, recs = counted(eng, lambda: eng.export_streams(ids, resampler=True))
        imp, _ = counted(eng, lambda: eng.import_streams(ids, recs))
        want = (0, 0) if n == 0 else (old_exp + 1, old_imp + 1)
        assert (exp, imp) == want, (eng.input_rate, n, old_exp, old_imp)
    assert n == 0 or old_exp >= 2
