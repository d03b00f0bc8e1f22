"""The playback guard on the H100 (include/mww.h, "playback guard").  Writes and reads are compared bit for bit with the NumPy
statement of the rule (tests/playback_guard_ref.py, itself checked against the g++ emulation of the header bodies in
tests/test_playback_guard.py); scores with a fresh StreamEngine of the same container over the reference clips read back,
then positive_scores; flags and passed with the CPU rule at every heard-rule edge:

- seeded write sequences at 4 096 streams with 512 rows and 65 536 streams with 4 096 rows, with releases as S advances,
  resets, and MWW_ENOMEM leaving the guard unchanged;
- the detector form against the streams form on the drained events, with 0, 1 and capacity events and the same launches,
  on a grouped detector and on model k of a MultiModelDetector;
- a synthetic self-wake: a stream whose own playback the model scores above the cutoff is flagged, one that only hears the
  same audio and one that played something else pass;
- the serving chain verify -> media guard -> playback guard -> endpointer arm;
- a move of streams between guards through heads, read and write at rebased starts, and state_dict."""

import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import playback_guard_ref as ref  # noqa: E402
from test_gpu_event_positions import F32, I8  # noqa: E402

from microwakeword_b200._lib import MwwError  # noqa: E402
from microwakeword_b200.detection import MultiModelDetector, StreamDetector, positive_scores  # noqa: E402
from microwakeword_b200.engine import MultiModelEngine, StreamEngine  # noqa: E402
from microwakeword_b200.playback import PlaybackGuard  # noqa: E402
from microwakeword_b200.synth_audio import synth_audio  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def advance(eng, calls, seed=0):
    """`calls` live calls of 480 samples of low noise on every stream"""
    rng = np.random.default_rng(seed)
    for _ in range(calls):
        eng.step(torch.from_numpy(rng.integers(-64, 64, (eng.n_streams, 480)).astype(np.int16)).to(DEV))
    torch.cuda.synchronize()


def same_reads(pb, model, ids, ends, n):
    got = pb.read(ids, ends, n).cpu().numpy()
    for i, (s, e) in enumerate(zip(ids, ends)):
        assert np.array_equal(got[i], model.read(int(s), int(e), n)), (i, s, e)


@pytest.mark.parametrize("n_streams, rows", [(4096, 512), (65536, 4096)])
def test_writes_and_reads_are_the_rule(n_streams, rows):
    rng = np.random.default_rng(n_streams)
    C = 4096
    eng = StreamEngine(F32, n_streams=n_streams)
    eng.set_audio_history(8000)
    pb = PlaybackGuard(F32, eng, slots=64, rows=rows, capacity_s=C / 16000, n_samples=1600, max_delay=800, window=1, ignore_steps=0)
    model = ref.Rule(n_streams, rows, C, lo=-(1 << 14), hi=1 << 17)
    streams = rng.choice(n_streams, rows + rows // 2, replace=False).astype(np.int32)
    for call in range(12):
        S = eng.audio_samples_seen
        k = int(rng.integers(rows // 8, rows // 2))
        ids = rng.choice(streams, k, replace=False).astype(np.int32)
        L = int(rng.choice([480, 1000, 3, 5000]))
        starts = S + rng.integers(-2000, 2000, k)
        if call % 3 == 0:
            starts -= starts % 8                     # the 8-sample vector form
        x = rng.integers(-32768, 32768, (k, L)).astype(np.int16)
        want = model.write(ids, starts, x, S)
        before = pb.heads()
        if want == ref.ENOMEM:
            with pytest.raises(MwwError) as e:
                pb.play(ids, torch.from_numpy(x).to(DEV) if call % 2 else x, starts=starts)
            assert e.value.code == -4
            assert all(np.array_equal(a, b) for a, b in zip(before, pb.heads()))
        else:
            pb.play(ids, torch.from_numpy(x).to(DEV) if call % 2 else x, starts=starts)
        rows_now, heads = pb.heads()
        assert {int(s): int(heads[s]) for s in np.flatnonzero(rows_now >= 0)} == model.head
        if call % 4 == 3:
            gone = rng.choice(streams, 16, replace=False).astype(np.int32)
            pb.reset(gone)
            model.reset(gone)
        probe = rng.choice(streams, 64, replace=False).astype(np.int32)
        same_reads(pb, model, probe, S + rng.integers(-3000, 3000, 64), int(rng.choice([800, 2400, 4096])))
        advance(eng, int(rng.integers(1, 6)), seed=call)
    assert pb.info().rows_used == len(model.head)


def fresh_scores(clips, window=5, ignore=25):
    fresh = StreamEngine(F32, n_streams=clips.shape[0])
    probs = fresh.predict_clip(clips.contiguous())
    return positive_scores(list(probs), window, ignore)


def test_scores_are_a_fresh_engine_and_flags_follow_the_rule_at_every_heard_edge():
    n = 64
    C, N, dmin, dmax = 32000, 8000, 160, 1760
    L = N + dmax - dmin
    eng = StreamEngine(F32, n_streams=n)
    eng.set_audio_history(16000)
    advance(eng, 60)
    S = eng.audio_samples_seen                                  # 28 800
    pb = PlaybackGuard(F32, eng, slots=n, rows=16, capacity_s=C / 16000, n_samples=N, min_delay=dmin, max_delay=dmax, ignore_steps=0,
                       cutoff=0.0)
    model = ref.Rule(n, 16, C, lo=-(1 << 15), hi=1 << 17)
    ids = np.arange(8, dtype=np.int32)
    x = np.stack([synth_audio(20000, 40 + s) for s in range(8)])
    starts = np.array([S - 21000] * 4 + [S - 12000] * 4, np.int64)
    pb.play(ids, x, starts=starts)
    model.write(ids, starts, x, S)
    w1, w2 = S - 1000, S + 8000                                 # S - C bounds streams 0-3, w - C streams 4-7
    r0 = np.array([S - C - 1, S - C, w1 - 1, w1, w2 - C - 1, w2 - C, w2 - 1, w2, S], np.int64)
    ends = r0 + dmin + L
    check_ids = np.array([0, 1, 2, 3, 4, 5, 6, 7, 40], np.int32)    # 40: no row
    conf = np.arange(10, 19, dtype=np.int32)
    scores, flagged, passed = (t.cpu().numpy() for t in pb.check(check_ids, confirmed=conf, ends=ends))
    clips = pb.read(check_ids, ends - dmin, L)
    want_scores = fresh_scores(clips, 5, 0)
    heard = [model.heard(int(s), int(r), S) for s, r in zip(check_ids, r0)]
    assert heard == [False, True, True, False, False, True, True, False, False]
    for i in range(9):
        ws, wf, wp = ref.decide(heard[i], want_scores[i], 0.0, int(conf[i]))
        assert (np.isnan(ws) and np.isnan(scores[i])) or scores[i] == ws, i
        assert (flagged[i], passed[i]) == (wf, wp), i
    assert flagged.any()
    # without confirmed ids a slot passes its own stream
    _, f2, p2 = (t.cpu().numpy() for t in pb.check(check_ids, ends=ends))
    assert np.array_equal(p2, np.where(f2 == 1, -1, check_ids)) and np.array_equal(f2, flagged)


GROUPED_EVENT = np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])


def live_loop(eng, dets, steps=40, n=512):
    shared = synth_audio(steps * 480, 11)
    for step in range(steps):
        chunk = np.stack([synth_audio(480, 100 * step + s) for s in range(8)] * (n // 8))
        chunk[: n // 2] = shared[step * 480:(step + 1) * 480]
        probs = eng.step(torch.from_numpy(chunk).to(DEV))
        for det in dets:
            det.update(probs) if hasattr(det, "roles") else det.update(probs, eng)
    torch.cuda.synchronize()


def same_as_check_streams(pb, eng, got, events, model, conf, post):
    S = eng.audio_samples_seen
    k = len(events)
    mine = np.ones(k, bool) if model is None else events["reserved"] == model
    ids = np.ascontiguousarray(events["stream"][mine], np.int32)
    t = [x.cpu().numpy() for x in pb.check(ids, confirmed=conf[:k][mine], ends=np.minimum(events["sample"][mine] + post, S))]
    assert np.array_equal(got[0][:k][mine], t[0], equal_nan=True)
    for g, w in zip(got[1:], t[1:]):
        assert np.array_equal(g[:k][mine], w)
    other = np.concatenate([np.flatnonzero(~mine), np.arange(k, len(got[0]))])
    assert np.isnan(got[0][other]).all() and (got[1][other] == 0).all() and np.array_equal(got[2][other], conf[other])
    return int(mine.sum())


def play_everyone(pb, eng, n, seed):
    """every other stream plays a seeded reply from a little before now"""
    ids = np.arange(0, n, 2, dtype=np.int32)[:pb.rows]
    x = np.stack([synth_audio(24000, seed + int(s)) for s in ids])
    pb.play(ids, x, starts=np.full(ids.size, eng.audio_samples_seen - 20000, np.int64))


def test_detector_form_is_check_streams_on_the_drained_events_with_the_same_launches_for_0_1_and_capacity_events():
    n, post, cap = 512, 3200, 64
    eng = StreamEngine(F32, n_streams=n)
    eng.set_audio_history(48000)
    full = StreamDetector(n, 0.05, capacity=cap, timed=True, groups=n // 2, group_window=1440)
    full.set_groups(np.arange(n), np.arange(n) // 2)
    one = StreamDetector(n, 0.05, capacity=cap, timed=True, groups=1, group_window=1 << 22)
    one.set_groups(np.arange(n), np.zeros(n, np.int32))
    pb = PlaybackGuard(F32, eng, slots=cap, rows=256, capacity_s=4.0, n_samples=16000, max_delay=3200, cutoff=0.0)
    conf = np.random.default_rng(3).integers(-1, n, cap).astype(np.int32)
    conf_d = torch.from_numpy(conf).to(DEV)

    def launches(det):
        before = pb.launch_count
        got = [t.cpu().numpy() for t in pb.check(det, conf_d, post=post)]
        return pb.launch_count - before, got

    per_call, got = launches(full)
    assert int(full.event_count.item()) == 0 and np.isnan(got[0]).all() and np.array_equal(got[2], conf)
    live_loop(eng, [full, one])
    play_everyone(pb, eng, n, 500)
    one.flush()
    assert int(one.event_count.item()) == 1 and int(full.event_count.item()) >= cap
    for det, k in ((one, 1), (full, cap)):
        calls, got = launches(det)
        assert calls == per_call
        events, m = det._drain_slots(GROUPED_EVENT)
        assert len(events) == k
        assert same_as_check_streams(pb, eng, got, events, None, conf, post) == k


def test_model_k_of_a_multi_model_detector_is_check_streams_on_its_events():
    n, post, cap = 512, 3200, 256
    eng = MultiModelEngine([F32, I8], n_streams=n)
    eng.set_audio_history(48000)
    mdet = MultiModelDetector(eng, [0.05, 0.05], capacity=cap, timed=True, groups=n // 2, group_window=1440)
    mdet.set_groups(np.arange(n), np.arange(n) // 2)
    live_loop(eng, [mdet])
    pb = PlaybackGuard(F32, eng, slots=cap, rows=256, capacity_s=4.0, n_samples=16000, max_delay=3200, cutoff=0.0)
    play_everyone(pb, eng, n, 900)
    conf = np.random.default_rng(4).integers(-1, n, cap).astype(np.int32)
    got = {k: [t.cpu().numpy() for t in pb.check(mdet, torch.from_numpy(conf).to(DEV), model=k, post=post)] for k in (0, 1)}
    events, m = mdet._drain_slots(GROUPED_EVENT)
    heard = [same_as_check_streams(pb, eng, got[k], events, k, conf, post) for k in (0, 1)]
    assert all(h >= 1 for h in heard) and sum(heard) == len(events), heard


def room(rng, x):
    taps = 48
    h = rng.normal(0, 1, taps) * np.exp(-np.arange(taps) / rng.uniform(4, 12)) * 0.4
    h[0] = 1.0
    return np.clip(np.round(rng.uniform(0.5, 1.2) * np.convolve(x.astype(np.float64), h)[:x.size]), -32768, 32767).astype(np.int16)


def self_wake_case(pad):
    """(the cutoff, a clip the model scores above it, one it scores below it): seeded synth_audio clips, each scored as the
    guard hears it, with `pad` zeros before and after (the reference window is wider than the clip by the delay spread)"""
    cand = np.stack([synth_audio(24000, 7000 + k) for k in range(64)])
    s = fresh_scores(torch.from_numpy(np.pad(cand, ((0, 0), (pad, pad)))).to(DEV))
    hi, lo = int(np.argmax(s)), int(np.argmin(s))
    cutoff = float(np.median(s))
    assert s[hi] > cutoff > s[lo], s
    return cutoff, cand[hi], cand[lo]


def test_a_device_that_says_the_wake_word_is_flagged_and_the_others_pass():
    """A plays a clip the model scores above the cutoff and hears it through a seeded room 2 400 samples later; B hears the same
    audio but played nothing; C played a clip the model scores below the cutoff"""
    rng = np.random.default_rng(12)
    n, A, B, Cs = 16, 3, 7, 11
    eng = StreamEngine(F32, n_streams=n)
    eng.set_audio_history(64000)
    advance(eng, 4)
    cutoff, loud, quiet = self_wake_case(1600)            # L_ref = 24000 + 4000 - 800: 1600 samples either side of a reply
    pb = PlaybackGuard(F32, eng, slots=8, rows=8, capacity_s=6.0, n_samples=24000, min_delay=800, max_delay=4000, cutoff=cutoff)
    S0 = eng.audio_samples_seen
    pb.play([A, Cs], np.stack([loud, quiet]))                    # starts=None: from now
    delay = 2400
    heard = np.zeros((n, 24000 + 4800), np.int16)
    mic = room(rng, np.concatenate([np.zeros(delay, np.int16), loud]))
    heard[A, :mic.size] = heard[B, :mic.size] = mic
    for k in range(heard.shape[1] // 480):
        eng.step(torch.from_numpy(heard[:, 480 * k:480 * (k + 1)].copy()).to(DEV))
    e = S0 + delay + 24000
    assert eng.audio_samples_seen >= e
    scores, flagged, passed = (t.cpu().numpy() for t in pb.check(np.array([A, B, Cs], np.int32), ends=np.full(3, e, np.int64)))
    assert list(flagged) == [1, 0, 0] and list(passed) == [-1, B, Cs], scores
    assert np.isnan(scores[1]) and scores[0] > cutoff > scores[2]


def test_serving_chain_arms_exactly_the_streams_that_pass_every_stage():
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.media import MediaGuard
    from microwakeword_b200.verify import Verifier
    n, post, cap = 512, 3200, 64
    eng = StreamEngine(F32, n_streams=n)
    eng.set_audio_history(48000)
    det = StreamDetector(n, 0.05, capacity=cap, timed=True)
    live_loop(eng, [det])
    ver = Verifier(F32, slots=cap, n_samples=16000, cutoff=0.0)
    guard = MediaGuard(slots=cap, n_samples=16000, ring=64, min_matches=1000)
    pb = PlaybackGuard(F32, eng, slots=cap, rows=256, capacity_s=4.0, n_samples=16000, max_delay=3200, cutoff=0.0)
    play_everyone(pb, eng, n, 300)
    ep = Endpointer(eng, capacity=cap)
    scores, confirmed = ver.verify(eng, det, at_event=True, post=post)
    _, _, gpassed = guard.check(eng, det, confirmed, post=post)
    pscores, flagged, passed = pb.check(det, gpassed, post=post)
    ep.arm(passed)
    torch.cuda.synchronize()
    want = set(passed.cpu().numpy().tolist()) - {-1}
    assert want and flagged.cpu().numpy().any()
    c, g, p, f = (t.cpu().numpy() for t in (confirmed, gpassed, passed, flagged))
    assert np.array_equal(p, np.where(f == 1, -1, g)) and np.array_equal(g, c)
    assert set(ep.armed_ids.cpu().numpy().tolist()) - {-1} == want


def test_a_move_between_guards_and_state_dict_give_equal_checks():
    n = 256
    eng = StreamEngine(F32, n_streams=n)
    eng.set_audio_history(32000)
    advance(eng, 20)
    kw = dict(slots=64, rows=64, capacity_s=3.0, n_samples=16000, max_delay=3200, cutoff=0.0)
    a = PlaybackGuard(F32, eng, **kw)
    ids = np.arange(0, 128, 3, dtype=np.int32)
    S = eng.audio_samples_seen
    a.play(ids, np.stack([synth_audio(30000, 60 + int(s)) for s in ids]), starts=S - 20000 + ids.astype(np.int64) * 37)
    a.play(ids[:10], np.stack([synth_audio(1000, 90 + int(s)) for s in ids[:10]]))
    ends = np.full(ids.size, S + 1500, np.int64)
    want = [t.cpu().numpy() for t in a.check(ids, ends=ends)]
    # move: heads and read on a, write on b at the starts that put each row back where it was on b's axis (the same axis here)
    b = PlaybackGuard(F32, eng, **kw)
    rows, heads = a.heads()
    C = a.capacity
    b.play(ids, a.read(ids, heads[ids], C), starts=heads[ids] - C)
    got = [t.cpu().numpy() for t in b.check(ids, ends=ends)]
    assert np.array_equal(got[0], want[0], equal_nan=True) and all(np.array_equal(g, w) for g, w in zip(got[1:], want[1:]))
    c = PlaybackGuard(F32, eng, **kw)
    c.load_state_dict(a.state_dict())
    got = [t.cpu().numpy() for t in c.check(ids, ends=ends)]
    assert np.array_equal(got[0], want[0], equal_nan=True) and all(np.array_equal(g, w) for g, w in zip(got[1:], want[1:]))
    assert not np.isnan(want[0]).all()
