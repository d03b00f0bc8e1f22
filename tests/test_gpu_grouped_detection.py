"""Grouped detection on the H100 (include/mww.h, "grouped detection").  Every grouped detector runs beside an ungrouped timed
twin on the same probabilities; the twin's events, fed through the NumPy rule (tests/detector_groups_ref.py) with each update's
clock and the groups of that update, must be the grouped detector's events exactly (stream, step, score bits, sample, group,
candidates), and the rows' state the twin's bit for bit:

- a 4 099-stream live loop on an fp32 engine, replayed at poll intervals D = 1, 7 and 33 (the same winners), twice (the same
  result), with groups changed mid-run, and with fired_ids / event_samples checked slot by slot against the drain;
- the anchored verify on the grouped detector against the independent path on the winners;
- a 65 536-row run of live and 100-step calls in uniform and per-row mode, 16 384 households of one to four rows;
- an int8 multi-model detector with two wake words and a VAD, merged per (group, model);
- two launches per grouped update with 0, 1 and many events; flush, state_dict round trip and refusals."""

import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from detector_groups_ref import GroupRule  # noqa: E402
from test_gpu_event_positions import (F32, I8, N, audio, captured_kernels, quantile_cutoff, reference_at,  # noqa: E402
                                      same, split)

from microwakeword_b200 import _lib  # noqa: E402
from microwakeword_b200.detection import MultiModelDetector, StreamDetector  # noqa: E402
from microwakeword_b200.engine import MultiModelEngine, StreamEngine  # noqa: E402
from microwakeword_b200.verify import Verifier  # noqa: E402

pytestmark = pytest.mark.gpu

WIN = 480


class Clock:
    """the counters of one engine call, as a timed plain detector's update reads them"""

    def __init__(self, eng=None, S=0, hop=160, buffered=320, stride=3, pending=0):
        if eng is not None:
            S, hop, buffered, stride, pending = eng.audio_samples_seen, eng.hop, eng.frontend_buffered, eng.stride, eng.pending_rows
        self.S, self.hop, self.frontend_buffered, self.stride, self.pending_rows = int(S), int(hop), int(buffered), int(stride), int(pending)

    def _audio_history(self):
        return 1, self.S

    def last_end(self):
        return self.S - (self.frontend_buffered - (WIN - self.hop)) - self.hop * self.pending_rows

    def step_samples(self):
        return self.hop * self.stride


def households(n_rows, n_groups, rng, ungrouped=0.1):
    """groups of one to four rows each for n_groups households over a random permutation of the rows; a share left at -1"""
    g = np.full(n_rows, -1, np.int32)
    perm, at = rng.permutation(n_rows), 0
    for h in range(n_groups):
        k = int(rng.integers(1, 5))
        g[perm[at:at + k]] = h
        at += k
        if at >= n_rows:
            break
    g[rng.random(n_rows) < ungrouped] = -1
    return g


def ev_key(e, model=None):
    return (int(e["group"]), -1 if model is None else int(model), int(e["stream"]), int(e["step"]), int(np.float32(e["score"]).view(np.uint32)),
            int(e["sample"]), int(e["candidates"]))


def rule_events(twin_events, updates, W):
    """the grouped events the rule gives: twin_events (timed, drained after every update, so list i holds update i's events),
    updates[i] = (a_u, E_u, groups at update i); plain detector (row = stream)"""
    ref, out = GroupRule(W), []
    for ev, (a, E, groups) in zip(twin_events, updates):
        cands = {}
        for e in ev:
            g = int(groups[e["stream"]])
            if g < 0:
                out.append(dict(stream=e["stream"], step=e["step"], score=e["score"], sample=e["sample"], group=-1, candidates=1))
            else:
                cands.setdefault(g, []).append(dict(stream=e["stream"], step=e["step"], score=e["score"], sample=e["sample"], row=e["stream"]))
        out += ref.update(cands, a, E)
    out += ref.flush()
    return sorted(ev_key(e) for e in out)


def same_rows(a, b):
    for k in ("hist", "seen", "cooldown"):
        assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), k


def check_slots(det):
    """fired_ids and event_samples slot by slot against the drain in slot order"""
    fired, pos = det.fired_ids.cpu().numpy().copy(), det.event_samples.cpu().numpy().copy()
    ev, n = det._drain_slots(np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)]))
    m = ev.size
    assert np.array_equal(fired[:m], ev["stream"]) and np.array_equal(pos[:m], ev["sample"]) and (fired[m:] == -1).all()
    return ev, n


def replay(calls, n_rows, cut, W, n_groups, group_plan, D=1, per_row=None, capacity=1 << 16, twin=False):
    """run a detector over recorded (probs, clock) calls; group_plan: {call index: groups from then on}.  -> (events as sorted
    keys, twin events per update or None, updates, final state)"""
    det = StreamDetector(n_rows, cut, capacity=capacity, timed=True, **({} if twin else dict(groups=n_groups, group_window=W)))
    if per_row is not None:
        det.set_cutoffs(per_row[0], per_row[1])
    groups = np.full(n_rows, -1, np.int32)
    got, per_update, updates = [], [], []
    for i, (p, clk) in enumerate(calls):
        if i in group_plan:
            groups = group_plan[i]
            if not twin:
                det.set_groups(np.arange(n_rows), groups)
        if p.shape[1] == 0:                                      # no step: no update
            continue
        det.update(p, clk)
        n = p.shape[1]
        updates.append((clk.last_end() - (n - 1) * clk.step_samples(), clk.last_end() + clk.step_samples(), groups.copy()))
        if twin:
            per_update.append(det.drain()[0])
        elif (i + 1) % D == 0:
            ev, n_ev = check_slots(det)
            assert n_ev == ev.size
            got += [ev_key(e) for e in ev]
    if not twin:
        det.flush()
        ev, _ = check_slots(det)
        got += [ev_key(e) for e in ev]
    state = det.state_dict()
    det.close()
    return sorted(got), per_update, updates, state


@pytest.fixture(scope="module")
def live_calls():
    """4 099 fp32 streams, 120 live calls: each call's probabilities and clock, recorded once"""
    S, n_calls = 4099, 120
    x = audio(S, 480 * n_calls, 41)
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(48000)
    calls = []
    for c in split(x, [480] * n_calls):
        p = eng.step(c)
        calls.append((p.clone(), Clock(eng)))
    cut = quantile_cutoff([p for p, _ in calls], 0.6)
    eng.close()
    return S, calls, cut, x


@pytest.mark.parametrize("W", [0, 4800])
def test_live_loop_is_the_rule_at_every_poll_interval(live_calls, W):
    S, calls, cut, _ = live_calls
    rng = np.random.default_rng(W)
    plan = {0: households(S, 1400, rng), 60: households(S, 1400, rng)}
    _, twin_ev, updates, twin_state = replay(calls, S, cut, W, 1400, plan, twin=True)
    want = rule_events(twin_ev, updates, W)
    assert len(want) > 50 and sum(k[-1] > 1 for k in want) > 5 and sum(k[0] < 0 for k in want) > 0
    runs = {}
    for D in (1, 7, 33, 7):
        got, _, _, state = replay(calls, S, cut, W, 1400, plan, D=D)
        assert got == want, D
        same_rows(state, twin_state)
        runs.setdefault(D, []).append(got)
    assert runs[7][0] == runs[7][1]


def test_anchored_verify_hears_the_winners(live_calls):
    S, calls, cut, x = live_calls
    xh = x.cpu().numpy()
    eng = StreamEngine(F32, n_streams=S)
    C = 48000
    eng.set_audio_history(C)
    det = StreamDetector(S, cut, capacity=4096, timed=True, groups=1400, group_window=3200)
    det.set_groups(np.arange(S), households(S, 1400, np.random.default_rng(3)))
    ver = Verifier(I8, slots=4096, n_samples=N, cutoff=0.5)
    post, checked = 3200, 0
    for i, c in enumerate(split(x, [480] * len(calls))):
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
        assert (ev["candidates"] >= 1).all()
    assert checked > 10
    ver.close()
    eng.close()


@pytest.mark.parametrize("per_row", [False, True])
def test_65536_rows_live_and_clip_calls(per_row):
    R, G, W = 65536, 16384, 2400
    rng = np.random.default_rng(7 + per_row)
    groups = households(R, G, rng)
    gen = torch.Generator(device="cuda").manual_seed(5)
    hh = torch.rand(G + 1, 1, device="cuda", generator=gen)
    gidx = torch.from_numpy(np.where(groups < 0, G, groups).astype(np.int64)).cuda()
    calls, S = [], 0
    for i, n in enumerate([1] * 40 + [100] + [1] * 30 + [100, 100] + [1] * 20):
        base = hh.expand(G + 1, n) if i % 2 else torch.rand(G + 1, n, device="cuda", generator=gen)
        p = (0.6 * base[gidx] + 0.4 * torch.rand(R, n, device="cuda", generator=gen)).contiguous()
        S += 480 * n
        calls.append((p, Clock(S=S)))
    cut = 0.8
    pr = (np.arange(0, R, 5), cut - 0.03) if per_row else None
    _, twin_ev, updates, twin_state = replay(calls, R, cut, W, G, {0: groups}, per_row=pr, capacity=1 << 21, twin=True)
    want = rule_events(twin_ev, updates, W)
    got, _, _, state = replay(calls, R, cut, W, G, {0: groups}, D=5, per_row=pr, capacity=1 << 21)
    assert len(want) > 1000 and sum(k[-1] > 1 for k in want) > 100
    assert got == want
    same_rows(state, twin_state)


def test_launches_flush_state_and_refusals():
    R = 512
    det = StreamDetector(R, 0.1, cooldown_slices=10, capacity=4096, timed=True, groups=100, group_window=2 ** 22)
    groups = np.where(np.arange(R) % 2 == 0, (np.arange(R) // 2) % 100, -1).astype(np.int32)      # odd rows ungrouped
    det.set_groups(np.arange(R), groups)
    assert (det.groups == groups).all()
    one = torch.zeros(R, 8)
    one[3, 2] = 1.0
    S, counts = 0, []
    for probs in (torch.zeros(R, 16), one, torch.ones(R, 60), torch.zeros(R, 8)):    # 0 events, 1 (row 3), many (warp form), many
        S += 480 * probs.shape[1]
        p = probs.cuda()
        before = int(det.event_count.item())
        assert captured_kernels(lambda: det.update(p, Clock(S=S))) == 2
        counts.append(int(det.event_count.item()) - before)
    assert counts[0] == 0 and counts[1] == 1 and counts[2] > 1
    torch.cuda.synchronize()
    st = det.state_dict()
    assert st["group_windows"]["open"].sum() > 0
    other = StreamDetector(R, 0.1, cooldown_slices=10, capacity=4096, timed=True, groups=100, group_window=2 ** 22)
    other.load_state_dict(st)
    same_rows(other.state_dict(), st)
    assert (other.groups == st["groups"]).all() and np.array_equal(other.group_windows(), st["group_windows"])
    n_open = int(st["group_windows"]["open"].sum())
    det.drain()
    assert captured_kernels(lambda: det.flush()) == 1
    ev, _ = det.drain()
    assert det.group_windows()["open"].sum() == 0 and ev.size == n_open and (ev["group"] >= 0).all() and (ev["candidates"] >= 1).all()
    # refusals leave the detector as it was
    with pytest.raises(_lib.MwwError, match="already grouped"):
        det._group(2, 0)
    for ids, g in (([R], [0]), ([0, 0], [1, 2]), ([0], [100]), ([0], [-2])):
        with pytest.raises(_lib.MwwError):
            det.set_groups(ids, g)
    assert (det.groups == groups).all()
    timed = StreamDetector(R, 0.5, timed=True)
    for n, w in ((0, 0), (R + 1, 0), (1, -1), (1, 2 ** 22 + 1)):
        with pytest.raises(_lib.MwwError):
            timed._group(n, w)
    timed.update(torch.ones(R, 8).cuda(), Clock(S=480 * 8))
    with pytest.raises(_lib.MwwError, match="may hold events"):
        timed._group(2, 0)
    with pytest.raises(ValueError, match="groups must be"):
        det.load_state_dict(dict(st, groups=st["groups"][:-1]))
    for d in (det, other, timed):
        d.close()


def test_models_detector_keeps_group_and_model_apart():
    Sm = 900
    sets = [np.arange(Sm), np.arange(0, Sm, 2), np.arange(Sm)]
    eng = MultiModelEngine([I8, I8, I8], n_streams=Sm, streams=sets)
    eng.set_audio_history(48000)
    sizes = [480] * 60 + [N] + [480] * 40
    x = audio(Sm, sum(sizes), 17)
    first = [torch.cat(p, 1) for p in zip(*[eng.predict_clip(c) for c in split(x, sizes)])]
    cut = [float(np.quantile(p.unfold(1, 5, 1).mean(2).amax(1).cpu().numpy(), 0.5)) for p in first]
    vad_cut = float(np.quantile(first[2].unfold(1, 5, 1).mean(2).cpu().numpy(), 0.1))
    eng.reset()
    eng.set_audio_history(48000)
    kw = dict(cutoffs=[cut[0], cut[1] - 0.02, vad_cut], vad=2, capacity=8192, timed=True)
    W = 2400
    twin, grp = MultiModelDetector(eng, **kw), MultiModelDetector(eng, groups=300, group_window=W, **kw)
    groups = households(Sm, 300, np.random.default_rng(9))
    grp.set_groups(np.arange(Sm), groups)
    ref, want, got = GroupRule(W), [], []
    hop = eng.hop
    for i, c in enumerate(split(x, sizes)):
        p = eng.predict_clip(c)
        twin.update(p)
        grp.update(p)
        row_end = eng.audio_samples_seen - (eng.frontend_buffered - (WIN - hop))
        after = eng.pending_rows
        a = {}
        cands = {}
        ev, _ = twin.drain()
        for k in (0, 1):
            n_k = p[k].shape[1]
            a_k = row_end - hop * (after[k] + (n_k - 1) * eng.stride[k]) if n_k else None
            for g in range(300):
                a[(g, k)] = a_k
        for e in ev:
            g = int(groups[e["stream"]])
            d = dict(stream=e["stream"], step=e["step"], score=e["score"], sample=e["sample"], row=e["stream"], model=e["model"])
            if g < 0:
                want.append(ev_key(dict(d, group=-1, candidates=1), e["model"]))
            else:
                cands.setdefault((g, int(e["model"])), []).append(d)
        want += [ev_key(dict(e, group=e["group"][0], candidates=e["candidates"]), e["group"][1]) for e in ref.update(cands, a, row_end + hop)]
        if i % 13 == 12:
            ev, _ = grp.drain()
            got += [ev_key(e, e["model"]) for e in ev]
    grp.flush()
    ev, _ = grp.drain()
    got += [ev_key(e, e["model"]) for e in ev]
    want += [ev_key(dict(e, group=e["group"][0], candidates=e["candidates"]), e["group"][1]) for e in ref.flush()]
    assert sorted(got) == sorted(want)
    assert len(want) > 20 and {k[1] for k in want} == {0, 1} and sum(k[-1] > 1 for k in want) > 3
    a, b = twin.state_dict(), grp.state_dict()
    for k in (0, 1, 2):
        for name in a["models"][k]:
            assert np.array_equal(a["models"][k][name].view(np.uint8), b["models"][k][name].view(np.uint8))
    for d in (twin, grp):
        d.close()
    eng.close()
