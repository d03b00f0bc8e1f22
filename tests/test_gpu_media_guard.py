"""The media guard on the H100 (include/mww.h, "media guard").  Every check is compared bit for bit with the CPU rule -- the
g++ emulation of the header bodies, itself checked against the NumPy statement in tests/test_media_guard.py -- applied to the
NumPy fingerprints of the feature rows that a fresh frontend gives from the audio read back from the engine's history:

- the device fingerprints (read back through the ring in state_dict) against the NumPy fingerprint of those rows;
- a synthetic broadcast through check_streams at 4 096 and 65 536 streams: one seeded advert heard by many households, each
  through its own gain, seeded exponential-decay room and 10-20 dB of independent noise, with 0-3 steps of onset jitter, among
  independent streams; then, on this synthetic data only, the broadcast slots are flagged and the independent ones are not;
- a registered clip that flags a lone household hearing a segment of it;
- the detector form against check_streams on the drained events, with 0, 1 and capacity events and the same launches each
  time, and model k of a grouped MultiModelDetector the same way;
- guards whose clips need more shared memory than the first one launched on the device;
- state_dict / load_state_dict: a new guard continues as the original does."""

import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import media_guard_ref as ref  # noqa: E402
from test_gpu_event_positions import F32  # noqa: E402
from test_media_guard import emul  # noqa: E402

from microwakeword_b200.detection import StreamDetector  # noqa: E402
from microwakeword_b200.engine import StreamEngine  # noqa: E402
from microwakeword_b200.media import MediaGuard  # noqa: E402
from microwakeword_b200.synth_audio import synth_audio  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
N = 24000


def features_of(clips):
    """the rows a fresh frontend emits from each clip [n, L] int16 (CUDA), as numpy [n, T, 40]"""
    fe = StreamEngine(None, n_streams=clips.shape[0])
    return fe.features(clips.contiguous()).cpu().numpy()


def cpu_rule(guard, eng, ids, ends, households, confirmed=None, ring_state=None, clips=()):
    """(matches, media, passed) of the emulated rule over the fingerprints of the clips read back from eng's history; the
    guard's ring as `ring_state` (a state_dict blob) before the call"""
    ids, ends = np.asarray(ids, np.int32), np.asarray(ends, np.int64)
    n, W, Ng = ids.size, guard.words, guard.n_samples
    S, C = eng.audio_samples_seen, eng.audio_history_capacity
    valid = (ids >= 0) & (ids < eng.n_streams) & (ends - Ng >= S - C)
    read = eng.audio_history(torch.from_numpy(np.where(valid, ids, -1).astype(np.int32)).to(DEV), Ng, end=torch.from_numpy(ends).to(DEV))
    fps = np.stack([ref.fingerprint(f) for f in features_of(read)])
    rid = np.where(valid, ids, -1).astype(np.int32)
    hh = np.full(n, -1, np.int32) if households is None else np.asarray(households, np.int32)
    r = guard.rule
    R = max(r.ring, 1)
    ring_fp, ring_pos = np.zeros((R, W), np.uint64), np.zeros(R, np.int64)
    ring_stream, ring_hh = np.zeros(R, np.int32), np.zeros(R, np.int32)
    count = np.zeros(1, np.int64)
    if ring_state is not None:
        b = ring_state
        count[0] = b[:8].view(np.int64)[0]
        o = 32
        ring_fp[:r.ring] = b[o:o + r.ring * W * 8].view(np.uint64).reshape(r.ring, W); o += r.ring * W * 8
        ring_pos[:r.ring] = b[o:o + r.ring * 8].view(np.int64); o += r.ring * 8
        ring_stream[:r.ring] = b[o:o + r.ring * 4].view(np.int32); o += r.ring * 4
        ring_hh[:r.ring] = b[o:o + r.ring * 4].view(np.int32)
    cfp = np.concatenate(clips) if len(clips) else np.zeros(1, np.uint64)
    clen = np.array([len(c) for c in clips] or [0], np.int32)
    conf = None if confirmed is None else np.ascontiguousarray(confirmed, np.int32)
    out = [np.zeros(n, np.int32) for _ in range(3)]
    fp = np.ascontiguousarray(fps, np.uint64)
    emul().emul_check(n, W, fp.ctypes.data, ids.ctypes.data, rid.ctypes.data, hh.ctypes.data, ends.ctypes.data,
                      None if conf is None else conf.ctypes.data, r.ring, count.ctypes.data, ring_fp.ctypes.data, ring_stream.ctypes.data,
                      ring_hh.ctypes.data, ring_pos.ctypes.data, len(clips), cfp.ctypes.data, clen.ctypes.data, r.max_lag, r.min_overlap,
                      r.max_ber_milli, r.min_matches, r.window_samples, *(o.ctypes.data for o in out))
    return out, fps


def room(rng, x):
    """x through a seeded exponential-decay FIR room with a gain"""
    taps = 48
    h = rng.normal(0, 1, taps) * np.exp(-np.arange(taps) / rng.uniform(4, 12)) * 0.4
    h[0] = 1.0
    return rng.uniform(0.3, 1.5) * np.convolve(x.astype(np.float64), h)[:x.size]


def with_noise(rng, x):
    snr = rng.uniform(10, 20)
    p = np.mean(x ** 2) + 1e-9
    return np.clip(np.round(x + rng.normal(0, np.sqrt(p / 10 ** (snr / 10)), x.size)), -32768, 32767).astype(np.int16)


def advert_audio(L, seed):
    """an advert of seeded synth_audio segments of 0.1 s: its level and tones change every 100 ms, as programme audio does
    (one long synth_audio is stationary noise, whose fingerprint 10 dB of room noise scrambles)"""
    return np.concatenate([synth_audio(1600, seed * 1000 + k) for k in range(-(-L // 1600))])[:L]


def broadcast_audio(n_streams, L, slots_b, slots_i, seed):
    """[n_streams, L] int16 on the device: the advert through a room, noise and 0-3 steps of onset jitter on slots_b, independent
    synth_audio streams on slots_i, silence elsewhere"""
    rng = np.random.default_rng(seed)
    advert = advert_audio(L, seed)
    x = torch.zeros((n_streams, L), dtype=torch.int16, device=DEV)
    rows = {}
    for s in slots_b:
        j = int(rng.integers(0, 4)) * 480
        a = np.concatenate([synth_audio(j, seed + 7)[:j], advert[:L - j]]) if j else advert
        rows[s] = with_noise(rng, room(rng, a))
    for k, s in enumerate(slots_i):
        rows[s] = synth_audio(L, 1000 * seed + k + 1)
    ids = np.array(sorted(rows), np.int64)
    x[torch.from_numpy(ids).to(DEV)] = torch.from_numpy(np.stack([rows[s] for s in ids])).to(DEV)
    return x


@pytest.mark.parametrize("n_streams", [4096, 65536])
def test_synthetic_broadcast_is_the_cpu_rule(n_streams):
    rng = np.random.default_rng(n_streams)
    L = N + 4 * 480
    eng = StreamEngine(None, n_streams=n_streams)
    eng.set_audio_history(32000)
    picked = rng.choice(n_streams, 160, replace=False).astype(np.int32)
    slots_b, slots_i = picked[:96], picked[96:]
    # seeds whose independent streams match no other stream: stationary synth_audio (a steady tone, noise near the frontend's
    # floor) has nearly constant rows, and two such clips share nearly all-zero fingerprints and match each other
    eng.features(broadcast_audio(n_streams, L, slots_b, slots_i, seed={4096: 3, 65536: 539}[n_streams]))
    S = eng.audio_samples_seen
    order = rng.permutation(picked.size)
    ids = picked[order]
    ends = np.full(ids.size, S, np.int64)
    households = np.arange(ids.size, dtype=np.int32)
    households[1] = households[0]                              # two satellites of one household
    guard = MediaGuard(slots=256, ring=64)
    got = [t.cpu().numpy() for t in guard.check(eng, ids, ends=ends, households=households)]
    want, _ = cpu_rule(guard, eng, ids, ends, households)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    is_b = np.isin(ids, slots_b)
    assert (got[1][is_b] & 2).all() and not got[1][~is_b].any(), (got[0][is_b], got[0][~is_b])
    assert (got[2][is_b] == -1).all() and np.array_equal(got[2][~is_b], ids[~is_b])
    # a second check of the same slots matches the ring too, and invalid slots pass their confirmed id
    state = guard.state_dict()["state"]
    ids2 = ids.copy()
    ids2[:3] = (-1, n_streams, ids[3])
    ends2 = ends.copy()
    ends2[3] = S - 32000 + N - 1                               # this clip has partly left the ring
    conf = rng.integers(-1, n_streams, ids.size).astype(np.int32)
    got = [t.cpu().numpy() for t in guard.check(eng, ids2, confirmed=conf, ends=ends2, households=households)]
    want, _ = cpu_rule(guard, eng, ids2, ends2, households, confirmed=conf, ring_state=state)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert list(got[0][:4]) == [-1, -1, got[0][2], -1] and list(got[2][[0, 1, 3]]) == list(conf[[0, 1, 3]])


def test_device_fingerprints_are_the_numpy_fingerprints_of_the_rows():
    eng = StreamEngine(None, n_streams=64)
    eng.set_audio_history(32000)
    eng.features(broadcast_audio(64, 30000, [], list(range(64)), seed=5))
    ids = np.arange(64, dtype=np.int32)
    ends = eng.audio_samples_seen - np.arange(64, dtype=np.int64) * 37
    guard = MediaGuard(slots=64, ring=64, min_matches=64)
    guard.check(eng, ids, ends=ends)
    _, fps = cpu_rule(guard, eng, ids, ends, None)
    b = guard.state_dict()["state"]
    W = guard.words
    assert b[:8].view(np.int64)[0] == 64
    assert np.array_equal(b[32:32 + 64 * W * 8].view(np.uint64).reshape(64, W), fps)


def test_registered_clip_flags_a_lone_household():
    rng = np.random.default_rng(9)
    advert = advert_audio(160000, 77)
    eng = StreamEngine(None, n_streams=8)
    eng.set_audio_history(32000)
    L = 30000
    x = torch.zeros((8, L), dtype=torch.int16, device=DEV)
    x[2] = torch.from_numpy(with_noise(rng, room(rng, advert[53123:53123 + L]))).to(DEV)
    x[5] = torch.from_numpy(synth_audio(L, 4)).to(DEV)
    eng.features(x)
    guard = MediaGuard(slots=8, ring=16, min_overlap=60)
    assert guard.register(advert) == 0
    assert guard.register(advert[:N // 2].astype(np.float32) / 32768.0) == 1        # shorter than the clip, float32 on the host
    ids, ends = np.array([2, 5], np.int32), np.full(2, eng.audio_samples_seen, np.int64)
    got = [t.cpu().numpy() for t in guard.check(eng, ids, ends=ends)]
    clips = [ref.fingerprint(f) for f in (features_of(torch.from_numpy(advert).to(DEV)[None])[0],
                                         features_of(torch.from_numpy(advert[:N // 2]).to(DEV)[None])[0])]
    want, _ = cpu_rule(guard, eng, ids, ends, None, clips=clips)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert got[1][0] & 1 and got[1][1] == 0 and list(got[2]) == [-1, 5]
    assert guard.info().n_media == 2
    guard.clear_registered()
    assert guard.info().n_media == 0


def live_loop(eng, dets, steps=40, n=512):
    """`steps` live calls: half the streams hear one broadcast, the rest eight independent sources; every detector updated"""
    shared = synth_audio(steps * 480, 11)
    for step in range(steps):
        chunk = np.stack([synth_audio(480, 100 * step + s) for s in range(8)] * (n // 8))
        chunk[: n // 2] = shared[step * 480:(step + 1) * 480]
        probs = eng.step(torch.from_numpy(chunk).to(DEV))
        for det in dets:
            det.update(probs) if hasattr(det, "roles") else det.update(probs, eng)
    torch.cuda.synchronize()


GROUPED_EVENT = np.dtype([("stream", np.int32), ("reserved", np.int32), ("step", np.int64), ("score", np.float32), ("pad", np.int32)])


def same_as_check_streams(eng, got, events, model, conf, post):
    """slot by slot (events in slot order, as drained): the detector form's results equal check_streams on the slots of
    `model` (None: every slot) with stream, end = min(P + post, S), household = group and the same confirmed ids; the other slots are unheard and pass
    their confirmed id.  (The detector form compares positions P, check_streams the ends; with the 60 s window every pair is in
    range either way.)"""
    S = eng.audio_samples_seen
    k = len(events)
    mine = np.ones(k, bool) if model is None else events["reserved"] == model
    twin = MediaGuard(slots=len(got[0]), ring=512, min_matches=2)
    ids = np.ascontiguousarray(events["stream"][mine], np.int32)
    t = [x.cpu().numpy() for x in twin.check(eng, ids, confirmed=conf[:k][mine], ends=np.minimum(events["sample"][mine] + post, S),
                                             households=events["group"][mine])]
    for g, w in zip(got, t):
        assert np.array_equal(g[:k][mine], w)
    other = np.concatenate([np.flatnonzero(~mine), np.arange(k, len(got[0]))])
    assert (got[0][other] == -1).all() and (got[1][other] == 0).all() and np.array_equal(got[2][other], conf[other])
    return int(mine.sum())


def test_detector_form_is_check_streams_on_the_drained_events_with_the_same_launches_for_0_1_and_capacity_events():
    n, post, cap = 512, 3200, 64
    eng = StreamEngine(F32, n_streams=n)
    eng.set_audio_history(48000)
    full = StreamDetector(n, 0.05, capacity=cap, timed=True, groups=n // 2, group_window=1440)
    full.set_groups(np.arange(n), np.arange(n) // 2)
    one = StreamDetector(n, 0.05, capacity=cap, timed=True, groups=1, group_window=1 << 22)   # one window: one event at flush
    one.set_groups(np.arange(n), np.zeros(n, np.int32))
    guard = MediaGuard(slots=cap, ring=512, min_matches=2)
    rng = np.random.default_rng(3)
    conf = rng.integers(-1, n, cap).astype(np.int32)
    conf_d = torch.from_numpy(conf).to(DEV)

    def launches(det):
        guard.clear_ring()                                      # as the check_streams twin's: each case hears only its own slots
        before = guard.launch_count
        got = [t.cpu().numpy() for t in guard.check(eng, det, conf_d, post=post)]
        return guard.launch_count - before, got

    per_call, got = launches(full)                              # no event yet
    assert int(full.event_count.item()) == 0 and (got[0] == -1).all() and np.array_equal(got[2], conf)
    live_loop(eng, [full, one])
    one.flush()
    assert int(one.event_count.item()) == 1 and int(full.event_count.item()) >= cap
    for det, k in ((one, 1), (full, cap)):
        calls, got = launches(det)
        assert calls == per_call
        events, m = det._drain_slots(GROUPED_EVENT)
        assert len(events) == k
        assert same_as_check_streams(eng, got, events, None, conf, post) == k


def test_model_k_of_a_grouped_multi_model_detector_is_check_streams_on_its_events():
    from microwakeword_b200.detection import MultiModelDetector
    from microwakeword_b200.engine import MultiModelEngine
    from test_gpu_event_positions import I8
    n, post, cap = 512, 3200, 256
    eng = MultiModelEngine([F32, I8], n_streams=n)
    eng.set_audio_history(48000)
    mdet = MultiModelDetector(eng, [0.05, 0.05], capacity=cap, timed=True, groups=n // 2, group_window=1440)
    mdet.set_groups(np.arange(n), np.arange(n) // 2)
    live_loop(eng, [mdet])
    conf = np.random.default_rng(4).integers(-1, n, cap).astype(np.int32)
    got = {k: [t.cpu().numpy() for t in MediaGuard(slots=cap, ring=512, min_matches=2).check(eng, mdet, torch.from_numpy(conf).to(DEV),
                                                                                               model=k, post=post)] for k in (0, 1)}
    events, m = mdet._drain_slots(GROUPED_EVENT)
    heard = [same_as_check_streams(eng, got[k], events, k, conf, post) for k in (0, 1)]
    assert all(h >= 1 for h in heard) and sum(heard) == len(events), heard


def test_guards_of_longer_clips_than_the_first_one_launched_still_run():
    """the match kernel's shared memory grows with the clip: above 48 KB from n_samples 100 640; a guard of 160 000 samples
    after one of 120 000 on the same device"""
    eng = StreamEngine(None, n_streams=8)
    eng.set_audio_history(160000)
    eng.features(broadcast_audio(8, 170000, [0, 1, 2, 3], [4, 5], seed=3))
    ids, ends = np.arange(6, dtype=np.int32), np.full(6, eng.audio_samples_seen, np.int64)
    for n_samples in (24000, 120000, 160000):
        guard = MediaGuard(slots=8, ring=8, n_samples=n_samples, max_media=0)
        got = [t.cpu().numpy() for t in guard.check(eng, ids, ends=ends)]
        want, _ = cpu_rule(guard, eng, ids, ends, None)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), n_samples


def test_state_dict_round_trip_continues_identically():
    rng = np.random.default_rng(21)
    eng = StreamEngine(None, n_streams=128)
    eng.set_audio_history(32000)
    slots_b, slots_i = np.arange(0, 40), np.arange(40, 80)
    eng.features(broadcast_audio(128, N + 1920, slots_b, slots_i, seed=31))
    ids = np.arange(80, dtype=np.int32)
    ends = np.full(80, eng.audio_samples_seen, np.int64)
    a = MediaGuard(slots=128, ring=100)
    a.register(synth_audio(50000, 8))
    a.check(eng, ids[:50], ends=ends[:50])
    b = MediaGuard(slots=128, ring=100)
    b.load_state_dict(a.state_dict())
    assert np.array_equal(b.state_dict()["state"], a.state_dict()["state"])
    perm = rng.permutation(80).astype(np.int32)
    for g1, g2 in zip(a.check(eng, perm, ends=ends), b.check(eng, perm, ends=ends)):
        assert torch.equal(g1, g2)
    assert np.array_equal(b.state_dict()["state"], a.state_dict()["state"])
    a.clear_ring()
    assert a.info().ring_count == 0 and b.info().ring_count == 130 and b.info().ring_fill == 100
