"""Group arbitration on the H100 (include/mww.h, "group arbitration").  Every arbitrated detector runs beside an ungrouped timed
twin on the same probabilities and the same engine.  The twin is drained right after each update, its events' levels are
computed in NumPy from eng.audio_history(ids, Ls + Ln, end=positions) read then, and the NumPy rule
(tests/group_arbitration_ref.py) must give the arbitrated detector's drained events exactly (stream, step, score bits, sample,
group, candidates, level bits), with the rows' state the twin's bit for bit:

- a 4 099-stream fp32 live loop in which each household's one to four streams hear one shared source at different gains over
  independent noise, at poll intervals 1, 7 and 33, with groups changed mid-run;
- households of a loud and a quiet copy of one voice: the loud copy wins, where the score-grouped detector picks the quiet one;
- 65 536 rows in 16 384 households, live and 100-step calls, uniform and per-row cutoffs;
- an int8 multi-model detector with two wake words and a VAD;
- the anchored verify on the winners; two launches per update with 0, 1 and many events; a non-default CUDA stream; the
  state_dict round trip; refusals."""

import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import group_arbitration_ref as ref  # noqa: E402
from test_gpu_event_positions import F32, I8, N, audio, captured_kernels, quantile_cutoff, reference_at, same, split  # noqa: E402
from test_gpu_grouped_detection import Clock, households, same_rows  # noqa: E402

from microwakeword_b200 import _lib  # noqa: E402
from microwakeword_b200.detection import MultiModelDetector, StreamDetector  # noqa: E402
from microwakeword_b200.engine import MultiModelEngine, StreamEngine  # noqa: E402
from microwakeword_b200.verify import Verifier  # noqa: E402

pytestmark = pytest.mark.gpu

LS, LN = 12000, 8000
C = 48000


def household_audio(groups, n_samples, seed, gains):
    """every stream of a household hears its household's source at its own gain, over independent noise; the source speaks in
    bursts of about 1 s, so that the spans before and during a burst differ"""
    S = groups.size
    src = audio(S, n_samples, seed).float()
    lead = np.arange(S)
    for g in np.unique(groups[groups >= 0]):
        members = np.flatnonzero(groups == g)
        lead[members] = members[0]
    gen = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.arange(n_samples, device="cuda")
    env = ((t // 16000) % 2 == 1).float() * 0.9 + 0.1
    x = src[torch.from_numpy(lead).cuda()] * env * torch.from_numpy(gains).cuda()[:, None].float()
    x += torch.randn(S, n_samples, device="cuda", generator=gen) * 150
    return x.clamp(-32768, 32767).to(torch.int16).contiguous()


def twin_levels(eng, ev):
    """the NumPy levels of drained events, from the history read now"""
    out = np.zeros(ev.size, np.float32)
    for i in range(0, ev.size, 8192):
        part = ev[i:i + 8192]
        a = eng.audio_history(part["stream"].astype(np.int32), LS + LN, end=part["sample"].astype(np.int64)).long()
        # the integer sums on the GPU (exact), the double arithmetic in NumPy
        sums = [t.cpu().numpy() for x in (a[:, LN:], a[:, :LN]) for t in ((x * x).sum(1), x.sum(1))]
        out[i:i + 8192] = ref.levels_from_sums(*sums, LS, LN)
    return out


def bits(x):
    x = np.float32(x)
    return -1 if np.isnan(x) else int(x.view(np.uint32))


def ev_key(e, model=-1):
    return (int(e["group"]), int(model), int(e["stream"]), int(e["step"]), bits(e["score"]), int(e["sample"]), int(e["candidates"]),
            bits(e["level"]))


class Twin:
    """the ungrouped timed twin of a plain detector and the NumPy rule over its events"""

    def __init__(self, n_rows, cut, W, per_row=None):
        self.det = StreamDetector(n_rows, cut, capacity=1 << 21, timed=True)
        if per_row is not None:
            self.det.set_cutoffs(*per_row)
        self.rule, self.want = ref.ArbRule(W), []

    def after_update(self, eng, n, groups):
        ev, _ = self.det.drain()
        lv = twin_levels(eng, ev)
        clk = Clock(eng)
        cands = {}
        for e, level in zip(ev, lv):
            g = int(groups[e["stream"]])
            d = dict(stream=e["stream"], step=e["step"], score=e["score"], sample=e["sample"], level=level, id=e["stream"])
            if g < 0:
                self.want.append(ev_key(dict(d, group=-1, candidates=1, level=np.nan)))
            else:
                cands.setdefault(g, []).append(d)
        self.want += [ev_key(e) for e in self.rule.update(cands, clk.last_end() - (n - 1) * clk.step_samples(), clk.last_end() + clk.step_samples())]

    def finish(self):
        self.want += [ev_key(e) for e in self.rule.flush()]
        return sorted(self.want)


def arbitrated(eng, n_rows, cut, G, W, per_row=None, **kw):
    det = StreamDetector(n_rows, cut, capacity=1 << 21, timed=True, groups=G, group_window=W)
    if per_row is not None:
        det.set_cutoffs(*per_row)
    det.arbitrate(eng, LS, LN, **kw)
    return det


def drain_keys(det):
    ev, n = det.drain()
    assert n == 0
    return [ev_key(e) for e in ev]


@pytest.fixture(scope="module")
def live():
    S, G, n_calls = 4099, 1400, 150
    rng = np.random.default_rng(11)
    plan = {0: households(S, G, rng), 75: households(S, G, rng)}
    gains = rng.uniform(0.2, 1.0, S).astype(np.float32)
    x = household_audio(plan[0], 480 * n_calls, 23, gains)
    eng = StreamEngine(F32, n_streams=S)
    probs = [eng.step(c).clone() for c in split(x, [480] * n_calls)]
    cut = quantile_cutoff(probs, 0.7)
    eng.close()
    return S, G, plan, gains, x, cut


def run_live(live, D, W=4800, plan=None):
    S, G, plan0, _, x, cut = live
    plan = plan0 if plan is None else plan
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    twin, det = Twin(S, cut, W), arbitrated(eng, S, cut, G, W)
    got, groups = [], plan[0]
    for i, c in enumerate(split(x, [480] * (x.shape[1] // 480))):
        if i in plan:
            groups = plan[i]
            det.set_groups(np.arange(S), groups)
        p = eng.step(c)
        if p.shape[1] == 0:
            continue
        twin.det.update(p, eng)
        det.update(p, eng)
        twin.after_update(eng, p.shape[1], groups)
        if (i + 1) % D == 0:
            got += drain_keys(det)
    det.flush()
    got += drain_keys(det)
    same_rows(det.state_dict(), twin.det.state_dict())
    for d in (det, twin.det):
        d.close()
    eng.close()
    return sorted(got), twin.finish()


def test_live_loop_is_the_rule_at_every_poll_interval(live):
    runs = [run_live(live, D) for D in (1, 7, 33)]
    want = runs[0][1]
    assert len(want) > 50 and sum(k[6] > 1 for k in want) > 5 and sum(k[0] < 0 for k in want) > 0
    for got, w in runs:
        assert w == want and got == want


def test_the_louder_copy_of_a_household_wins():
    """households of two copies of one voice over equal independent noise, the louder copy on the higher row: both fire at the
    same step with the same score, so the score-grouped detector answers with the lower (quieter) row and the arbitrated one
    with the louder"""
    H, n = 512, 480 * 70
    R = 2 * H
    eng = StreamEngine(F32, n_streams=R)
    eng.set_audio_history(C)
    gen = torch.Generator(device="cuda").manual_seed(3)
    voice = torch.randn(H, n, device="cuda", generator=gen) * 3000
    voice[:, :n - 6000] = 0                                   # the voice speaks in the last 6 000 samples only
    gain = torch.tensor([0.3, 1.0], device="cuda").repeat(H)[:, None]
    x = (voice.repeat_interleave(2, 0) * gain + torch.randn(R, n, device="cuda", generator=gen) * 300).clamp(-32768, 32767).to(torch.int16)
    for c in split(x, [480] * 70):
        eng.step(c)
    kw = dict(window=1, cooldown_slices=0, timed=True, groups=H, group_window=0)
    score, arb = StreamDetector(R, 0.5, **kw), StreamDetector(R, 0.5, **kw)
    for d in (score, arb):
        d.set_groups(np.arange(R), np.arange(R) // 2)
    arb.arbitrate(eng, 4000, 8000)
    p = torch.ones(R, 1, device="cuda")
    score.update(p, eng)
    arb.update(p, eng)
    (es, _), (ea, _) = score.drain(), arb.drain()
    assert es.size == ea.size == H and (ea["candidates"] == 2).all()
    assert (es["stream"] % 2 == 0).all() and (ea["stream"] % 2 == 1).all()
    quiet = StreamDetector(R, 0.5, window=1, cooldown_slices=0, timed=True)
    quiet.update(p, eng)
    ev, _ = quiet.drain()
    a = eng.audio_history(ev["stream"].astype(np.int32), 12000, end=ev["sample"].astype(np.int64)).cpu().numpy()
    lv = ref.levels_of(a, 4000, 8000)
    assert np.array_equal(ea["level"].view(np.uint32), lv[1::2].view(np.uint32)) and (lv[1::2] > lv[0::2]).all()
    for d in (score, arb, quiet):
        d.close()
    eng.close()


@pytest.mark.parametrize("per_row", [False, True])
def test_65536_rows_live_and_100_step_calls(per_row):
    R, G, W = 65536, 16384, 2400
    rng = np.random.default_rng(7 + per_row)
    groups = households(R, G, rng)
    eng = StreamEngine(F32, n_streams=R)
    eng.set_audio_history(C)
    x = audio(1021, 480 * 40, 5)[torch.arange(R, device="cuda") % 1021].contiguous()
    gen = torch.Generator(device="cuda").manual_seed(5)
    hh = torch.rand(G + 1, 1, device="cuda", generator=gen)
    gidx = torch.from_numpy(np.where(groups < 0, G, groups).astype(np.int64)).cuda()
    cut = 0.8
    pr = (np.arange(0, R, 5), cut - 0.03) if per_row else None
    twin, det = Twin(R, cut, W, pr), arbitrated(eng, R, cut, G, W, pr)
    det.set_groups(np.arange(R), groups)
    got = []
    for i, c in enumerate(split(x, [480] * 40)):
        eng.step(c)
        n = 100 if i in (20, 30, 31) else 1
        base = hh.expand(G + 1, n) if i % 2 else torch.rand(G + 1, n, device="cuda", generator=gen)
        p = (0.6 * base[gidx] + 0.4 * torch.rand(R, n, device="cuda", generator=gen)).contiguous()
        twin.det.update(p, eng)
        det.update(p, eng)
        twin.after_update(eng, n, groups)
        if i % 5 == 4:
            got += drain_keys(det)
    det.flush()
    got += drain_keys(det)
    want = twin.finish()
    assert len(want) > 1000 and sum(k[6] > 1 for k in want) > 100
    assert sorted(got) == want
    same_rows(det.state_dict(), twin.det.state_dict())
    for d in (det, twin.det):
        d.close()
    eng.close()


def test_models_detector_with_two_wake_words_and_a_vad():
    Sm, G, W = 900, 300, 2400
    sets = [np.arange(Sm), np.arange(0, Sm, 2), np.arange(Sm)]
    eng = MultiModelEngine([I8, I8, I8], n_streams=Sm, streams=sets)
    eng.set_audio_history(C)
    sizes = [480] * 60 + [N] + [480] * 40
    groups = households(Sm, G, np.random.default_rng(9))
    x = household_audio(groups, sum(sizes), 17, np.random.default_rng(4).uniform(0.2, 1.0, Sm).astype(np.float32))
    first = [torch.cat(p, 1) for p in zip(*[eng.predict_clip(c) for c in split(x, sizes)])]
    cut = [float(np.quantile(p.unfold(1, 5, 1).mean(2).amax(1).cpu().numpy(), 0.5)) for p in first]
    vad_cut = float(np.quantile(first[2].unfold(1, 5, 1).mean(2).cpu().numpy(), 0.1))
    eng.reset()
    eng.set_audio_history(C)
    kw = dict(cutoffs=[cut[0], cut[1] - 0.02, vad_cut], vad=2, capacity=8192, timed=True)
    twin, det = MultiModelDetector(eng, **kw), MultiModelDetector(eng, groups=G, group_window=W, **kw)
    det.set_groups(np.arange(Sm), groups)
    det.arbitrate(eng, LS, LN)
    rule, want, got = ref.ArbRule(W), [], []
    hop = eng.hop
    for i, c in enumerate(split(x, sizes)):
        p = eng.predict_clip(c)
        twin.update(p)
        det.update(p)
        row_end = eng.audio_samples_seen - (eng.frontend_buffered - (480 - hop))
        after = eng.pending_rows
        ev, _ = twin.drain()
        lv = twin_levels(eng, ev)
        a, cands = {}, {}
        for k in (0, 1):
            n_k = p[k].shape[1]
            for g in range(G):
                a[(g, k)] = row_end - hop * (after[k] + (n_k - 1) * eng.stride[k]) if n_k else None
        for e, level in zip(ev, lv):
            g = int(groups[e["stream"]])
            d = dict(stream=e["stream"], step=e["step"], score=e["score"], sample=e["sample"], level=level, id=e["stream"])
            if g < 0:
                want.append(ev_key(dict(d, group=-1, candidates=1, level=np.nan), e["model"]))
            else:
                cands.setdefault((g, int(e["model"])), []).append(d)
        want += [ev_key(dict(e, group=e["group"][0]), e["group"][1]) for e in rule.update(cands, a, row_end + hop)]
        if i % 13 == 12:
            ev, _ = det.drain()
            got += [ev_key(e, e["model"]) for e in ev]
    det.flush()
    ev, _ = det.drain()
    got += [ev_key(e, e["model"]) for e in ev]
    want += [ev_key(dict(e, group=e["group"][0]), e["group"][1]) for e in rule.flush()]
    assert sorted(got) == sorted(want)
    assert len(want) > 20 and {k[1] for k in want} == {0, 1} and sum(k[6] > 1 for k in want) > 3
    for d in (twin, det):
        d.close()
    eng.close()


def test_anchored_verify_hears_the_winners(live):
    S, G, plan, _, x, cut = live
    xh = x.cpu().numpy()
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    det = StreamDetector(S, cut, capacity=4096, timed=True, groups=G, group_window=3200)
    det.arbitrate(eng, LS, LN)
    det.set_groups(np.arange(S), plan[0])
    ver = Verifier(I8, slots=4096, n_samples=N, cutoff=0.5)
    post, checked = 3200, 0
    for i, c in enumerate(split(x, [480] * (x.shape[1] // 480))):
        det.update(eng.step(c), eng)
        if i % 9 != 8:
            continue
        Sn = eng.audio_samples_seen
        ids, pos = det.fired_ids.cpu().numpy().copy(), det.event_samples.cpu().numpy()
        e = np.minimum(pos + post, Sn)
        ids[(ids >= 0) & (e - N < Sn - C)] = -1
        got = ver.verify(eng, det, at_event=True, post=post)
        same(got, reference_at(xh, ids, np.where(ids >= 0, e, -1), I8))
        checked += int((ids >= 0).sum())
        ev, _ = det.drain()
        assert (np.isnan(ev["level"]) == (ev["group"] < 0)).all()
    assert checked > 10
    ver.close()
    det.close()
    eng.close()


def test_launches_stream_state_and_refusals():
    R = 512
    eng = StreamEngine(F32, n_streams=R)
    eng.set_audio_history(C)
    x = audio(R, 480 * 8, 3)
    det = StreamDetector(R, 0.1, cooldown_slices=10, capacity=4096, timed=True, groups=100, group_window=2 ** 22)
    groups = np.where(np.arange(R) % 2 == 0, (np.arange(R) // 2) % 100, -1).astype(np.int32)
    det.set_groups(np.arange(R), groups)
    det.arbitrate(eng)
    assert (det.speech_samples, det.noise_samples) == (12000, 8000)
    one = torch.zeros(R, 8)
    one[4, 2] = 1.0
    counts = []
    for i, probs in enumerate((torch.zeros(R, 16), one, torch.ones(R, 60), torch.zeros(R, 8))):    # 0, 1 (row 4), many (warp form)
        eng.step(x[:, 480 * i:480 * (i + 1)].contiguous())
        p = probs.cuda()
        before = int(det.event_count.item())
        assert captured_kernels(lambda: det.update(p, eng)) == 2
        counts.append(int(det.event_count.item()) - before)
    assert counts[0] == 0 and counts[1] == 0 and counts[2] > 1                        # row 4 is grouped: its event waits in a window
    torch.cuda.synchronize()
    st = det.state_dict()
    assert st["group_windows"]["open"].sum() > 0 and (st["group_levels"][st["group_windows"]["open"] == 1] > 0).all()
    other = StreamDetector(R, 0.1, cooldown_slices=10, capacity=4096, timed=True, groups=100, group_window=2 ** 22)
    other.arbitrate(eng)
    other.load_state_dict(st)
    assert np.array_equal(other.group_levels().view(np.uint32), st["group_levels"].view(np.uint32))
    assert np.array_equal(other.group_windows(), st["group_windows"])
    det.drain()
    assert captured_kernels(lambda: det.flush()) == 1
    other.drain()
    other.flush()
    a, b = det.drain()[0], other.drain()[0]
    assert a.size == int(st["group_windows"]["open"].sum()) and a.tobytes() == b.tobytes() and np.isfinite(a["level"]).all()
    # a non-default CUDA stream: the update and the drain are ordered on it
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        eng.step(x[:, :480].contiguous())
        det.update(torch.ones(R, 40, device="cuda"), eng)
        det.flush()
        ev, _ = det.drain()
    assert ev.size > 0
    # refusals
    with pytest.raises(_lib.MwwError, match="already arbitrated"):
        det.arbitrate(eng)
    with pytest.raises(ValueError, match="bound"):
        det.update(torch.ones(R, 1, device="cuda"), StreamEngine(F32, n_streams=R))
    fresh = lambda: StreamDetector(R, 0.1, timed=True, groups=4, group_window=0)   # noqa: E731
    for s_, n_ in ((479, 8000), (12000, 479), ((1 << 20) + 1, 8000), (40000, 9000)):
        with pytest.raises(_lib.MwwError):
            fresh().arbitrate(eng, s_, n_)
    small = StreamEngine(F32, n_streams=R - 1)
    small.set_audio_history(C)
    with pytest.raises(_lib.MwwError, match="streams"):
        fresh().arbitrate(small)
    with pytest.raises(ValueError, match="groups"):
        StreamDetector(R, 0.1, timed=True).arbitrate(eng)
    busy = fresh()
    busy.update(torch.ones(R, 8, device="cuda"), eng)
    with pytest.raises(_lib.MwwError, match="may hold events"):
        busy.arbitrate(eng)
    shrink = fresh()
    shrink.arbitrate(eng)
    eng.set_audio_history(16000)
    with pytest.raises(_lib.MwwError, match="audio history"):
        shrink.update(torch.ones(R, 1, device="cuda"), eng)
    with pytest.raises(ValueError, match="group_levels"):
        det.load_state_dict({k: v for k, v in st.items() if k != "group_levels"})
    for d in (det, other, busy, shrink):
        d.close()
    eng.close()
