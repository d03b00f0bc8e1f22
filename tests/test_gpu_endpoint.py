"""Endpointing on the H100 (mww_endpointer_*; microwakeword_b200.endpoint.Endpointer) against tests/endpoint_ref.py: a
65 536-stream engine with audio history takes live and clip calls, the endpointer is fed controlled speech probabilities of
the calls' real step counts and placed by the handle's real counters, and its events, state, armed_ids and ended_ids equal
the reference exactly; the speech flags equal a models detector's VAD `active`; arming from a detector's fired_ids and a
verifier's confirmed ids on the device; command clips against the engine's own history reads, at 16 kHz, 48 kHz and G.711;
launch counts that depend on neither n nor how many rows are armed; and every refusal of the C-ABI on a live handle, which
leaves the endpointer's state and launch count unchanged."""

import os

import numpy as np
import pytest

import endpoint_ref as R
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")


def _probs(rng, rows, n, offset):
    """square waves of random period and phase per row, plus noise: speech runs and pauses"""
    period = rng.integers(4, 40, rows)[:, None]
    phase = rng.integers(0, 80, rows)[:, None]
    j = np.arange(offset, offset + n)[None, :]
    base = np.where(((j + phase) // period) % 2 == 0, 0.85, 0.1)
    return np.clip(base + rng.normal(0, 0.2, (rows, n)), 0, 1).astype(np.float32)


def _counters(eng):
    """the handle's counters an update is placed by: samples_seen, frontend_buffered and model 0's pending rows"""
    return eng.audio_samples_seen, int(eng._info().frontend_buffered), int(eng.pending_rows)


def _check_same(ep, ref, capacity):
    import torch
    torch.cuda.synchronize()
    got = ep.state_dict()
    want = ref.state()
    for k in ("hist", "seen", "flags", "armed", "elapsed", "run", "silence", "heard", "start_sample", "speech_end_sample", "positions"):
        assert np.array_equal(np.asarray(got[k]).astype(np.float64 if k == "hist" else np.int64) if k != "flags" else got[k],
                              np.asarray(want[k]).astype(np.float64 if k == "hist" else np.int64) if k != "flags" else want[k]), k
    for k in ("samples_seen", "buffered", "pending", "steps"):
        assert got[k] == want[k], k
    assert np.array_equal(ep.armed_ids.cpu().numpy(), ref.armed_ids())
    ended = ep.ended_ids.cpu().numpy()
    want_ended = ref.ended_ids()
    assert np.array_equal(np.sort(ended), np.sort(want_ended))


def _sorted(ev):
    ev = np.asarray(ev, R.EVENT)
    return ev[np.lexsort((ev["stream"], ev["end_sample"]))]


def test_65536_streams_live_and_clip_calls_match_the_reference():
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S, C = 65536, 32000
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    rule = dict(vad_window=5, vad_cutoff=0.5, speech_steps=3, silence_steps=8, timeout_steps=30, max_steps=60, lookback_steps=12)
    ep = Endpointer(eng, capacity=8192, **rule)
    ref = R.EndpointRef(S, np.arange(S), eng.stride, eng.hop, capacity=8192, counters=_counters(eng), **rule)
    rng = np.random.default_rng(0)
    gen = torch.Generator(device="cuda").manual_seed(1)
    used = 0
    calls = [480] * 12 + [4000, 1237, 480, 480, 9600] + [480] * 20 + [16000] + [480] * 10
    ep_launches = []
    for c, n16 in enumerate(calls):
        audio = (torch.randint(-3000, 3000, (S, n16), generator=gen, device="cuda", dtype=torch.int32)).to(torch.int16)
        probs = eng.predict_clip(audio)
        n = probs.shape[1]
        fake = _probs(rng, S, n, used)
        used += n
        before = ep.launch_count
        launches_before = eng.launch_count
        ep.update(torch.from_numpy(fake).cuda())
        assert eng.launch_count == launches_before                    # nothing launched on the handle
        ep_launches.append(ep.launch_count - before)
        ref.update(fake, *_counters(eng))
        if c in (3, 15, 30):
            ids = rng.choice(S, 3000 if c != 15 else 50, replace=False).astype(np.int32)
            b = ep.launch_count
            ep.arm(ids)
            assert ep.launch_count - b == 1
            ref.arm(ids)
        if c == 20:
            dev = torch.from_numpy(np.concatenate([rng.choice(S, 500), [-1, -1, S, S + 5]]).astype(np.int32)).cuda()
            ep.arm(dev)
            ref.arm(dev.cpu().numpy())
        if c == 25:
            ids = rng.choice(S, 400, replace=False)
            ep.disarm(ids)
            ref.disarm(ids)
            ep.reset(ids[:100])
            ref.reset(ids[:100])
        if c % 9 == 8:
            _check_same(ep, ref, 8192)
            (ge, gn), (re_, rn) = ep.drain(), ref.drain()
            assert gn == 0 and np.array_equal(_sorted(ge), _sorted(re_))
    assert set(ep_launches) == {1}
    _check_same(ep, ref, 8192)
    (ge, _), (re_, rn) = ep.drain(), ref.drain()
    assert np.array_equal(_sorted(ge), _sorted(re_))


def test_speech_flags_equal_the_models_detectors_vad_on_a_stream_subset():
    import torch
    from microwakeword_b200.detection import MultiModelDetector
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import MultiModelEngine
    S = 4096
    subset = np.arange(0, S, 3, dtype=np.int32)
    eng = MultiModelEngine([F32, F32], n_streams=S, streams=[None, subset])
    eng.set_audio_history(4800)
    det = MultiModelDetector(eng, cutoffs=[0.99, 0.3], windows=[5, 4], vad=1)
    ep = Endpointer(eng, model=1, vad_window=4, vad_cutoff=0.3)
    assert ep.n_rows == subset.size
    gen = torch.Generator(device="cuda").manual_seed(2)
    for n16 in [480] * 20 + [3000, 480, 777] + [480] * 10:
        audio = torch.randint(-8000, 8000, (S, n16), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        probs = eng.predict_clip(audio)
        det.update(probs)
        ep.update(probs[1])
        active = det.state_dict()["models"][1]["active"]
        flags = ep.state_dict()["flags"]
        assert np.array_equal((flags & np.uint64(1)).astype(np.int32), active)


def test_arming_from_device_lists_matches_host_arming():
    import torch
    from microwakeword_b200.detection import StreamDetector
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    from microwakeword_b200.verify import Verifier
    S = 2048
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(32000)
    eps = [Endpointer(eng, lookback_steps=10, capacity=S) for _ in range(3)]
    ver = Verifier(F32, slots=S, n_samples=16000, cutoff=-1.0)
    gen = torch.Generator(device="cuda").manual_seed(3)
    rng = np.random.default_rng(3)
    for _ in range(40):
        audio = torch.randint(-8000, 8000, (S, 480), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        probs = eng.step(audio)
        fake = torch.from_numpy(_probs(rng, S, probs.shape[1], 0)).cuda()
        for ep in eps:
            ep.update(fake)
    # a detector that fired on every 7th stream: fired_ids holds them in some order, then -1 in the unused slots
    det = StreamDetector(S, cutoff=0.5, window=1, cooldown_slices=0, capacity=S)
    p = torch.zeros((S, 1), dtype=torch.float32, device="cuda")
    p[::7] = 1.0
    det.update(p)
    fired = det.fired_ids                                      # the detector's own buffer, before its drain
    host = np.arange(0, S, 7, dtype=np.int32)
    got = fired.cpu().numpy()
    assert np.array_equal(np.sort(got[got >= 0]), host) and (got[host.size:] == -1).all()
    _, confirmed = ver.verify(eng, fired)                      # cutoff -1: every listed stream is confirmed, -1 elsewhere
    assert np.array_equal(np.sort(confirmed.cpu().numpy()[confirmed.cpu().numpy() >= 0]), host)
    eps[0].arm(fired)
    eps[1].arm(confirmed)
    eps[2].arm(host)
    torch.cuda.synchronize()
    states = [ep.state_dict() for ep in eps]
    for s in states[:2]:
        for k in ("armed", "elapsed", "run", "silence", "heard", "start_sample", "speech_end_sample"):
            assert np.array_equal(s[k], states[2][k]), k
    assert sorted(eps[2].armed_ids.cpu().numpy()[eps[2].armed_ids.cpu().numpy() >= 0].tolist()) == sorted(host.tolist())


def _commands_case(eng, ep, step_fn, calls, C, pre, post, max_samples):
    import torch
    rng = np.random.default_rng(5)
    S = eng.n_streams
    ids = np.arange(0, S, 2, dtype=np.int32)
    for c in range(calls):
        probs = step_fn(c)
        n = probs.shape[1]
        fake = torch.from_numpy(np.where(rng.random((S, n)) < 0.8, 0.9, 0.05).astype(np.float32)).cuda()
        if c < 20:
            fake[:] = 0.9                                       # speech first, then mostly speech: commands end on every reason
        ep.update(fake)
        if c == 2:
            ep.arm(ids)
    clips, lengths = ep.commands(pre=pre, post=post, max_samples=max_samples)
    hist = eng.audio_history(np.arange(S, dtype=np.int32), C)
    torch.cuda.synchronize()
    seen = eng.audio_samples_seen
    events, n = ep._drain_slots()
    assert n > 0
    h = hist.cpu().numpy()
    want, wl = R.commands(events, n, ep.capacity, pre, post, max_samples, seen, C, lambda s: h[s])
    assert np.array_equal(lengths.cpu().numpy(), wl)
    assert np.array_equal(clips.cpu().numpy(), want)
    return events, wl


@pytest.mark.parametrize("kind", ["pcm16", "48k", "ulaw"])
def test_command_clips_are_slices_of_the_history(kind):
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S, C = 256, 9600
    eng = StreamEngine(F32, n_streams=S, input_rate=48000 if kind == "48k" else 16000)
    eng.set_audio_history(C)
    ep = Endpointer(eng, speech_steps=2, silence_steps=4, timeout_steps=200, max_steps=50, lookback_steps=2, capacity=S)
    gen = torch.Generator(device="cuda").manual_seed(6)
    per_call = 1440 if kind == "48k" else 480

    def step(c):
        if kind == "ulaw":
            audio = torch.randint(0, 256, (S, per_call), generator=gen, device="cuda", dtype=torch.int32).to(torch.uint8)
            return eng.step(audio, law="ulaw")
        audio = torch.randint(-8000, 8000, (S, per_call), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        return eng.step(audio)

    # the commands run up to 50 steps = 24 000 samples, more than the 9 600 the ring keeps: their beginnings are zeros
    events, lengths = _commands_case(eng, ep, step, 90, C, pre=800, post=1600, max_samples=30000)
    assert set(events["reason"].tolist()) >= {R.MAX_LENGTH}
    assert (lengths > C).any()


def test_launch_counts_do_not_depend_on_n_or_armed_rows():
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S = 1024
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(48000)
    ep = Endpointer(eng, capacity=64)
    gen = torch.Generator(device="cuda").manual_seed(7)
    per = []
    for k, n16 in enumerate([480, 480, 4800, 480, 16000, 160, 480]):
        audio = torch.randint(-8000, 8000, (S, n16), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)
        probs = eng.predict_clip(audio)
        if k == 3:
            ep.arm(np.arange(S))
        h0, e0 = eng.launch_count, ep.launch_count
        ep.update(probs)
        per.append((probs.shape[1], eng.launch_count - h0, ep.launch_count - e0))
    assert {p[1] for p in per} == {0} and {p[2] for p in per} == {1}
    assert len({p[0] for p in per}) > 2
    e0 = ep.launch_count
    ep.commands(max_samples=4800)
    ep.arm(np.arange(10))
    ep.disarm(np.arange(5))
    ep.reset(np.arange(3))
    ep.reset()
    assert ep.launch_count - e0 == 5


def test_c_refusals_on_a_live_handle_leave_everything_unchanged():
    """each mww_endpointer_* refusal, called through the C-ABI with a live handle: MWW_EINVAL, a message, and the endpointer's
    state and launch count as they were"""
    import ctypes
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    L = _lib.lib()
    vp = ctypes.c_void_p
    S = 64

    def rule(**kw):
        r = dict(vad_window=5, speech_steps=3, silence_steps=25, timeout_steps=100, max_steps=334, lookback_steps=64, vad_cutoff=0.5)
        r.update(kw)
        return _lib.MwwEndpointRule(r["vad_window"], r["speech_steps"], r["silence_steps"], r["timeout_steps"], r["max_steps"],
                                    r["lookback_steps"], r["vad_cutoff"])

    def refused(rc, words):
        msg = L.mww_last_error(None)
        assert rc == -1 and msg and words in msg.decode(), (rc, msg, words)

    eng = StreamEngine(F32, n_streams=S)
    out = vp(1)
    refused(L.mww_endpointer_create(eng._h, 0, ctypes.byref(rule()), 4, ctypes.byref(out)), "no audio history")
    assert out.value is None
    eng.set_audio_history(9600)
    front = StreamEngine(None, n_streams=S)
    front.set_audio_history(9600)
    refused(L.mww_endpointer_create(front._h, 0, ctypes.byref(rule()), 4, ctypes.byref(out)), "frontend-only")
    for k in (-1, 1):
        refused(L.mww_endpointer_create(eng._h, k, ctypes.byref(rule()), 4, ctypes.byref(out)), "model")
    multi = MultiModelEngine([F32, F32], n_streams=S)
    multi.set_audio_history(9600)
    refused(L.mww_endpointer_create(multi._h, 2, ctypes.byref(rule()), 4, ctypes.byref(out)), "model 2")
    for kw, words in ((dict(vad_window=0), "vad_window"), (dict(vad_window=33), "vad_window"), (dict(vad_cutoff=float("nan")), "vad_cutoff"),
                      (dict(vad_cutoff=float("inf")), "vad_cutoff"), (dict(speech_steps=0), "speech_steps"), (dict(silence_steps=0), "silence_steps"),
                      (dict(timeout_steps=0), "timeout_steps"), (dict(max_steps=0), "max_steps"), (dict(lookback_steps=-1), "lookback_steps"),
                      (dict(lookback_steps=65), "lookback_steps")):
        refused(L.mww_endpointer_create(eng._h, 0, ctypes.byref(rule(**kw)), 4, ctypes.byref(out)), words)
        assert out.value is None
    refused(L.mww_endpointer_create(eng._h, 0, ctypes.byref(rule()), 0, ctypes.byref(out)), "capacity")

    ep = Endpointer(eng, capacity=4, timeout_steps=3)
    gen = torch.Generator(device="cuda").manual_seed(8)
    for _ in range(6):
        ep.update(eng.step(torch.randint(-8000, 8000, (S, 480), generator=gen, device="cuda", dtype=torch.int32).to(torch.int16)))
    ep.arm(np.arange(0, S, 2))
    torch.cuda.synchronize()
    before, launches, h_launches = ep.state_dict(), ep.launch_count, eng.launch_count

    def unchanged():
        after = ep.state_dict()
        assert after.keys() == before.keys()
        assert all(np.array_equal(np.asarray(after[k]), np.asarray(before[k])) for k in after)
        assert ep.launch_count == launches

    st = vp(torch.cuda.current_stream().cuda_stream)
    probs = torch.rand((S, 3), device="cuda")
    # a skipped update: the handle ran two one-step calls and the endpointer is told of one
    for _ in range(2):
        eng.step(torch.zeros((S, 480), dtype=torch.int16, device="cuda"))
    h_launches = eng.launch_count
    for n in (1, 3, 0):
        refused(L.mww_endpointer_update(ep._ep, probs.data_ptr(), n, 3, st), "do not match")
    refused(L.mww_endpointer_update(ep._ep, probs.data_ptr(), -1, 3, st), "n >= 0")
    refused(L.mww_endpointer_update(ep._ep, probs.data_ptr(), 2, 1, st), "pitch >= n")
    refused(L.mww_endpointer_update(ep._ep, None, 1, 1, st), "probabilities")
    unchanged()
    # the command read
    clips = torch.empty((4, 4800), dtype=torch.int16, device="cuda")
    lengths = torch.empty(4, dtype=torch.int32, device="cuda")
    other = StreamEngine(F32, n_streams=S)
    other.set_audio_history(9600)
    args = lambda h=eng._h, pre=0, post=0, m=4800, o=clips.data_ptr(), stride=4800, l=lengths.data_ptr(): (ep._ep, h, pre, post, m, o, stride, l, st)
    refused(L.mww_endpointer_read_commands(*args(h=other._h)), "not the one")
    refused(L.mww_endpointer_read_commands(*args(pre=-1)), "pre and post")
    refused(L.mww_endpointer_read_commands(*args(post=-1)), "pre and post")
    refused(L.mww_endpointer_read_commands(*args(m=-1, stride=0)), "max_samples")
    refused(L.mww_endpointer_read_commands(*args(m=(1 << 22) + 1, stride=(1 << 22) + 1)), "max_samples")
    refused(L.mww_endpointer_read_commands(*args(stride=4799)), "out_stride")
    refused(L.mww_endpointer_read_commands(*args(o=None)), "NULL output")
    refused(L.mww_endpointer_read_commands(*args(l=None)), "NULL output")
    unchanged()
    # host id lists and the drain
    bad = np.array([0, S], np.int32)
    for name in ("mww_endpointer_arm", "mww_endpointer_disarm", "mww_endpointer_reset"):
        refused(getattr(L, name)(ep._ep, bad.ctypes.data, 2, st), "out of range")
        refused(getattr(L, name)(ep._ep, bad.ctypes.data, -1, st), "n >= 0")
    for name in ("mww_endpointer_arm_device", "mww_endpointer_reset_device"):
        refused(getattr(L, name)(ep._ep, None, 3, st), "n >= 0")
    refused(L.mww_endpointer_drain(ep._ep, None, 4, None, st), "max_events")
    unchanged()
    # set_state: each bad field alone, the rest as get_state gave it
    for field, value, words in (("seen", -1, "negative seen"), ("elapsed", -1, "negative count"), ("run", -2, "negative count"),
                                ("silence", -3, "negative count"), ("heard", 2, "heard"), ("armed", 5, "armed"),
                                ("samples_seen", -1, "baseline"), ("buffered", 480, "baseline"), ("pending", 3, "baseline"),
                                ("steps", -1, "baseline")):
        d = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in before.items()}
        if isinstance(d[field], np.ndarray):
            d[field][0] = value
        else:
            d[field] = value
        with pytest.raises(_lib.MwwError) as e:
            ep.load_state_dict(d)
        assert e.value.args and words in str(e.value), (field, str(e.value))
        unchanged()
    assert eng.launch_count == h_launches                                               # no refusal launched on the handle
