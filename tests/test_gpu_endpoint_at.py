"""The positioned arm of the endpointer on the H100 (mww_endpointer_arm_at; Endpointer.arm(ids, at=...)) against
tests/endpoint_at_ref.py: a 65 536-stream engine with audio history takes live and clip calls with controlled speech
probabilities, and arm_at from host and device lists gives the reference's events, state, mute words, armed_ids and ended_ids
exactly, with launch counts that depend on neither n nor the armed rows; the pause after the wake word, which plain arm ends
on and the positioned arm carries through to the command, with the clip against the engine's own history read; timed plain,
grouped and models detectors on real engine probabilities; and a stream moved mid-mute between two handles, plain records
into a positioned endpointer, and the state_dict round trip."""

import os

import numpy as np
import pytest

import endpoint_ref as R
from conftest import GOLDEN
from endpoint_at_ref import PLACED, EndpointAtRef
from test_gpu_endpoint import _check_same, _counters, _probs, _sorted

pytestmark = pytest.mark.gpu

F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")


def _check_mutes(ep, ref):
    assert np.array_equal(ep.mutes(), ref.mute_words())


def test_65536_streams_arm_at_from_host_and_device_lists_matches_the_reference():
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S, C, CAP = 65536, 32000, 16384
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    rule = dict(vad_window=5, vad_cutoff=0.5, speech_steps=3, silence_steps=8, timeout_steps=30, max_steps=60, lookback_steps=12)
    ep = Endpointer(eng, capacity=CAP, **rule)
    ref = EndpointAtRef(S, np.arange(S), eng.stride, eng.hop, capacity=CAP, counters=_counters(eng), **rule)
    step = eng.stride * eng.hop
    rng = np.random.default_rng(0)
    gen = torch.Generator(device="cuda").manual_seed(1)
    used, launches, muted, placed = 0, {}, 0, 0
    calls = [480] * 12 + [4000, 1237, 480, 480, 9600] + [480] * 20 + [16000] + [480] * 10
    for c, n16 in enumerate(calls):
        audio = torch.randint(-3000, 3000, (S, n16), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        probs = eng.predict_clip(audio)
        n = probs.shape[1]
        fake = _probs(rng, S, n, used)
        used += n
        b = ep.launch_count
        ep.update(torch.from_numpy(fake).cuda())
        launches.setdefault("update", set()).add(ep.launch_count - b)
        ref.update(fake, *_counters(eng))
        q = ref.q()
        if c == 3:                                               # before the switch: the plain launches
            ids = rng.choice(S, 2000, replace=False).astype(np.int32)
            b = ep.launch_count
            ep.arm(ids)
            assert ep.launch_count - b == 1 and not ep.positioned
            ref.arm(ids)
        if c in (8, 15, 30):                                     # host lists, repeats at other positions, skips of every size
            k = 3000 if c != 15 else 40
            ids = rng.choice(S, k).astype(np.int32)
            pos = q - rng.integers(-3 * step, 16 * step, k)
            skip = {8: 5 * step + 17, 15: 0, 30: step}[c]
            b = ep.launch_count
            ep.arm(ids, at=pos.tolist(), skip=skip)
            launches.setdefault("arm_at", set()).add(ep.launch_count - b)
            ref.arm_at(ids, pos, skip)
        if c in (20, 33):                                        # device lists with -1 and out-of-range slots
            ids = np.concatenate([rng.choice(S, 1500), [-1, -1, S, S + 5]]).astype(np.int32)
            pos = (q - rng.integers(-2 * step, 14 * step, ids.size)).astype(np.int64)
            b = ep.launch_count
            ep.arm(torch.from_numpy(ids).cuda(), at=torch.from_numpy(pos).cuda(), skip=2 * step)
            launches.setdefault("arm_at", set()).add(ep.launch_count - b)
            ref.arm_at(ids, pos, 2 * step)
        if c == 25:
            ids = rng.choice(S, 400, replace=False)
            ep.arm(ids[:100])
            ref.arm(ids[:100])
            ep.disarm(ids[100:300])
            ref.disarm(ids[100:300])
            ep.reset(ids[300:])
            ref.reset(ids[300:])
        if c % 9 == 8:
            _check_same(ep, ref, CAP)
            _check_mutes(ep, ref)
            muted += int(((ref.mute_words() & (PLACED - 1)) > 0).sum())
            placed += int(((ref.mute_words() & PLACED) > 0).sum())
            (ge, gn), (re_, rn) = ep._drain_slots(), ref.drain()
            assert gn == rn and np.array_equal(_sorted(ge), _sorted(re_))
    assert ep.positioned and launches == {"update": {1}, "arm_at": {2}}
    assert muted > 100 and placed > 100 and (ref.state()["armed"] >= 0).sum() > 100   # running mutes and placed rows were checked
    _check_same(ep, ref, CAP)
    _check_mutes(ep, ref)
    (ge, gn), (re_, rn) = ep._drain_slots(), ref.drain()
    assert gn == rn > 0 and np.array_equal(_sorted(ge), _sorted(re_))


def test_launch_counts_do_not_depend_on_n_or_armed_rows():
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S = 1024
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(9600)
    ep = Endpointer(eng, capacity=S)
    gen = torch.Generator(device="cuda").manual_seed(4)
    for n in (0, 1, 5, S, 4 * S):
        audio = torch.randint(-8000, 8000, (S, 1440), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        probs = eng.step(audio)
        ids = torch.randint(-1, S + 2, (n,), generator=gen, device="cuda", dtype=torch.int32)
        pos = torch.full((n,), eng.audio_samples_seen, dtype=torch.int64, device="cuda") - 480 * torch.randint(0, 9, (n,), generator=gen,
                                                                                                              device="cuda")
        host = np.arange(min(n, S), dtype=np.int32)
        for fn, want in ((lambda: ep.update(torch.full_like(probs, 0.9)), 1), (lambda: ep.arm(ids, at=pos), 2),
                         (lambda: ep.arm(host, at=[eng.audio_samples_seen] * host.size, skip=0), 2), (lambda: ep.arm(ids), 1),
                         (lambda: ep.disarm(host[:3]), 1), (lambda: ep.reset(host[3:]), 1)):
            b = ep.launch_count
            fn()
            assert ep.launch_count - b == want
        assert ep.positioned


def _pause_run(arm_kind, silence_steps=20):
    """a 1 s wake word, the detection at its end (P), a 1.2 s pause, a 2 s command, then silence, in 30 ms live calls on
    4 streams; the VAD probabilities follow the script.  -> (events, clips, lengths, P, history reads of the commands)"""
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S = 4
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(16000 * 8)
    ep = Endpointer(eng, silence_steps=silence_steps, timeout_steps=200, max_steps=400, lookback_steps=64, capacity=S)
    script = [0.05] * 20 + [0.95] * 33 + [0.05] * 40 + [0.95] * 67 + [0.05] * 60      # 30 ms steps
    gen = torch.Generator(device="cuda").manual_seed(7)
    P = None
    for j, v in enumerate(script):
        audio = torch.randint(-8000, 8000, (S, 480), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        probs = eng.step(audio)
        ep.update(torch.full((S, probs.shape[1]), v, dtype=torch.float32, device="cuda"))
        if j == 52:                                         # the wake word's last step: the detector's position
            P = eng.audio_samples_seen
        if j == 60:                                         # the detection reaches the endpointer 8 steps later
            ids = torch.arange(S, dtype=torch.int32, device="cuda")
            if arm_kind == "plain":
                ep.arm(ids)
            else:
                ep.arm(ids, at=torch.full((S,), P, dtype=torch.int64, device="cuda"))
    clips, lengths = ep.commands(pre=0, post=3200, max_samples=16000 * 6)
    torch.cuda.synchronize()
    events, n = ep._drain_slots()
    ends = torch.from_numpy(np.minimum(events["speech_end_sample"] + 3200, events["end_sample"])).cuda()
    L = int(lengths.max().item())
    want = eng.audio_history(torch.from_numpy(events["stream"].copy()).cuda(), L, end=ends)
    return events, clips[:n, :L], lengths[:n], P, want


def test_a_pause_after_the_wake_word_ends_plain_arm_but_not_the_positioned_arm():
    ev, _, _, P, _ = _pause_run("plain")
    assert (ev["reason"] == R.END_OF_SPEECH).all() and ev.size == 4
    assert (ev["speech_end_sample"] <= P + 480 * 3).all() and (ev["start_sample"] < P - 16000 * 0.9).all()   # the wake word was the command
    ev, clips, lengths, P, want = _pause_run("at")
    assert (ev["reason"] == R.END_OF_SPEECH).all() and ev.size == 4
    assert (ev["start_sample"] == P).all()
    assert (ev["speech_end_sample"] >= P + 16000 * 3).all()                    # after the 1.2 s pause and the 2 s command
    # the clip is [P - pre, speech_end + post) of the history: the engine's own read that ends there
    assert (lengths.cpu().numpy() == (np.minimum(ev["speech_end_sample"] + 3200, ev["end_sample"]) - P)).all()
    assert lengths.min().item() == lengths.max().item()
    assert np.array_equal(clips.cpu().numpy(), want.cpu().numpy())


def _engine_run(eng, calls, gen, fn):
    import torch
    for c in range(calls):
        audio = (torch.randn((eng.n_streams, 480), generator=gen, device="cuda") * 6000).clamp(-32768, 32767).to(torch.int16)
        fn(c, eng.step(audio))


@pytest.mark.parametrize("kind", ["plain", "grouped", "models"])
def test_arm_at_a_detector_equals_arm_at_with_its_drained_positions(kind):
    import torch
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    S = 2048
    gen = torch.Generator(device="cuda").manual_seed(11)
    if kind == "models":
        eng = MultiModelEngine([F32, F32], n_streams=S)
        eng.set_audio_history(32000)
        det = MultiModelDetector(eng, cutoffs=[-1.0, -1.0], windows=[1, 1], cooldown_slices=[10, 10], capacity=8 * S,
                                 timed=True)
    else:
        eng = StreamEngine(F32, n_streams=S)
        eng.set_audio_history(32000)
        det = StreamDetector(S, cutoff=-1.0, window=1, cooldown_slices=10, capacity=8 * S, timed=True,
                             groups=S // 4 if kind == "grouped" else None, group_window=480 * 3 if kind == "grouped" else 0)
        if kind == "grouped":
            det.set_groups(np.arange(S), np.arange(S) // 4)
    eps = [Endpointer(eng, lookback_steps=40, capacity=8 * S) for _ in range(2)]
    fired = []

    def step(c, probs):
        if kind == "models":
            det.update(probs)
        else:
            det.update(probs, eng)
        for ep in eps:
            ep.update(probs[0] if kind == "models" else probs)
        if c in (30, 45):
            eps[0].arm(det.fired_ids, at=det)
            torch.cuda.synchronize()
            ev, _ = det.drain()
            fired.append(ev.size)
            eps[1].arm(ev["stream"].astype(np.int32), at=ev["sample"].astype(np.int64))
    _engine_run(eng, 60, gen, step)
    assert min(fired) > 0
    a, b = (ep.state_dict() for ep in eps)
    for k in ("armed", "elapsed", "run", "silence", "heard", "start_sample", "speech_end_sample", "mute"):
        assert np.array_equal(a[k], b[k]), k
    assert (a["armed"] >= 0).any()
    ea, eb = (ep.drain()[0] for ep in eps)
    assert np.array_equal(ea, eb)


def test_a_stream_moved_mid_mute_ends_as_if_it_had_stayed_and_checkpoints_round_trip():
    import torch
    from microwakeword_b200.endpoint import Endpointer, EndpointerRecords
    from microwakeword_b200.engine import StreamEngine
    S, C = 512, 48000
    rule = dict(silence_steps=6, timeout_steps=80, max_steps=200, lookback_steps=30)
    src, dst = StreamEngine(F32, n_streams=S), StreamEngine(F32, n_streams=S)
    for e in (src, dst):
        e.set_audio_history(C)
    ep, dep = Endpointer(src, capacity=S, **rule), Endpointer(dst, capacity=S, **rule)
    gen = torch.Generator(device="cuda").manual_seed(5)
    rng = np.random.default_rng(5)
    probs = _probs(rng, S, 200, 0)
    for c in range(50):                                   # the destination runs on its own first: a younger axis after the move
        pr = dst.step(torch.zeros((S, 480), dtype=torch.int16, device="cuda"))
        dep.update(torch.rand((S, pr.shape[1]), device="cuda") * 0.3)
    used = 0
    for c in range(80):
        pr = src.step(torch.randint(-8000, 8000, (S, 480), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16))
        n = pr.shape[1]
        ep.update(torch.from_numpy(probs[:, used:used + n]).cuda())
        used += n
    step = ep.stride * ep.hop
    q = src.audio_samples_seen - (int(src._info().frontend_buffered) - (480 - ep.hop)) - ep.hop * int(src.pending_rows)
    ids = np.arange(S, dtype=np.int32)
    ep.arm(ids, at=(q - step * (ids % 7)).tolist(), skip=step * 9)
    assert (ep.mutes() & (PLACED - 1)).any()
    # checkpoint round trip: into a fresh endpointer of the same engine
    st = ep.state_dict()
    twin = Endpointer(src, capacity=S, **rule)
    twin.load_state_dict(st)
    assert twin.positioned and all(np.array_equal(np.asarray(st[k]), np.asarray(twin.state_dict()[k])) for k in st)
    plain = {k: v for k, v in st.items() if k != "mute"}
    twin2 = Endpointer(src, capacity=S, **rule)
    twin2.load_state_dict(plain)
    assert not twin2.positioned and not twin2.mutes().any()
    # the move: history, and endpointer rows as positioned records (pad 1)
    dst.import_streams(ids, src.export_streams(ids, history=C))
    recs = ep.export_streams(ids)
    assert recs.layout.pad == 1 and not dep.positioned
    path = os.path.join(os.environ.get("TMPDIR", "/tmp"), "mww_endpoint_at_records_%d.npz" % os.getpid())
    recs.save(path)
    recs = EndpointerRecords.load(path, torch.device("cuda", 0))
    os.unlink(path)
    dep.import_streams(ids, recs)
    assert dep.positioned and np.array_equal(dep.mutes(), ep.mutes())
    shift = dst.audio_samples_seen - src.audio_samples_seen
    for c in range(80, 150):
        a = torch.randint(-8000, 8000, (S, 480), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        pr, prd = src.step(a), dst.step(a)
        n = pr.shape[1]
        p = torch.from_numpy(probs[:, used:used + n]).cuda()
        used += n
        ep.update(p)
        dep.update(p)
    clips, lens = ep.commands(pre=800, post=1600, max_samples=C)
    dclips, dlens = dep.commands(pre=800, post=1600, max_samples=C)
    torch.cuda.synchronize()
    ev, n = ep._drain_slots()
    dev_, dn = dep._drain_slots()
    assert n == dn > S // 2
    order, dorder = np.argsort(ev["stream"]), np.argsort(dev_["stream"])
    m = ev[order].copy()
    for k in ("start_sample", "end_sample", "speech_end_sample"):
        m[k] += shift
    assert np.array_equal(m, dev_[dorder])
    assert torch.equal(lens[torch.from_numpy(order).cuda()], dlens[torch.from_numpy(dorder).cuda()])
    assert torch.equal(clips[torch.from_numpy(order).cuda()], dclips[torch.from_numpy(dorder).cuda()])
    # plain records into a positioned endpointer: every mute word 0
    plain_ep = Endpointer(src, capacity=S, **rule)
    prec = plain_ep.export_streams(ids)
    assert prec.layout.pad == 0
    dep.import_streams(ids, prec)
    assert not dep.mutes().any()


def test_python_refusals_of_mixed_host_and_device_lists():
    import torch
    from microwakeword_b200.detection import StreamDetector
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    eng = StreamEngine(F32, n_streams=64)
    eng.set_audio_history(9600)
    ep = Endpointer(eng, capacity=64)
    dids = torch.zeros(4, dtype=torch.int32, device="cuda")
    dpos = torch.zeros(4, dtype=torch.int64, device="cuda")
    for kw, msg in ((dict(ids=[0, 1, 2, 3], at=dpos), "both"), (dict(ids=dids, at=[0, 0, 0, 0]), "both"),
                    (dict(ids=dids, at=dpos[:3]), "length"), (dict(ids=dids, at=dpos.to(torch.int32)), "int64"),
                    (dict(ids=dids.long(), at=dpos), "int32"), (dict(ids=dids, at=StreamDetector(64, 0.5, capacity=4)), "timed")):
        with pytest.raises(ValueError, match=msg):
            ep.arm(**kw)
    assert not ep.positioned and ep.launch_count == 0
