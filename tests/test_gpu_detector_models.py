"""The multi-model streaming detector on the GPU (run with -m gpu on an H100): MultiModelDetector behind a MultiModelEngine of
fp32 okay_nabu, int8 okay_nabu and the int8 run-time geometry of stride 17 (tests/generic_range.py's long_stride) as the VAD,
against the NumPy reference (tests/detector_models_ref.py) run on exactly the probabilities the engine returned: the same
event set with scores bit for bit, and the final state bit for bit.  30 ms live calls mixed with clip calls of other
lengths, so the models' steps and pending rows drift apart; 4 096 and 65 536 streams (past the first wave), with and
without stream sets; without a VAD against K StreamDetectors; the fired-id list restarting the streams that fired; state
moved to a second detector; and refusals that leave the state unchanged."""

import ctypes
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from detector_models_ref import OFF, VAD, WAKE, ModelsRef, same_model_events, same_model_state
from detector_ref import same_events, same_state
from generic_range import GEOMETRIES, models as range_models

pytestmark = pytest.mark.gpu

WIN_WAKE, WIN_VAD, COOLDOWN = 5, 3, 10


def _blobs():
    from microwakeword_b200 import model_file as MF
    f32, i8 = (open(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % k), "rb").read() for k in ("f32", "int8"))
    return [f32, i8, MF.write_container(range_models(GEOMETRIES["long_stride"])[1])]


def _sets(S, on, seed=3):
    if not on:
        return None
    rng = np.random.default_rng(seed)
    return [None, np.flatnonzero(rng.random(S) < 0.6).astype(np.int32), np.flatnonzero(rng.random(S) < 0.7).astype(np.int32)]


class Feed:
    """one engine, a pool of audio on the device and a seeded schedule of call lengths: 30 ms live calls and clip calls"""

    def __init__(self, torch, S, sets, seed):
        sys.path.insert(0, ROOT)
        from bench import synth_audio_device
        from microwakeword_b200.engine import MultiModelEngine
        self.torch = torch
        dev = torch.device("cuda", 0)
        self.eng = MultiModelEngine(_blobs(), S, streams=sets)
        self.pool = [synth_audio_device(torch, S, 4800, seed + i, dev) for i in range(3)]
        self.rng = np.random.default_rng(seed)
        self.i = 0

    def call(self):
        n = 480 if self.rng.random() < 0.75 else int(self.rng.choice([160, 800, 1440, 3200, 4800]))
        audio = self.pool[self.i % len(self.pool)][:, :n]
        self.i += 1
        pending = self.eng.pending_rows
        probs = self.eng.step(audio) if n == 480 else self.eng.predict_clip(audio)
        return probs, pending


def _cutoffs(torch, feed, calls=40):
    """cutoffs from the probabilities of `calls` calls: a wake cutoff that about a fifth of the streams' best averages
    exceed, and a VAD cutoff at the median average, so the flag turns on and off"""
    got = [[], [], []]
    for _ in range(calls):
        probs, _ = feed.call()
        for k, p in enumerate(probs):
            got[k].append(p)
    out = []
    for k, w in zip(range(3), (WIN_WAKE, WIN_WAKE, WIN_VAD)):
        p = torch.cat(got[k], 1)
        avg = p.unfold(1, w, 1).mean(-1)
        q = avg.max(1).values.quantile(0.8) if k < 2 else avg.flatten()[::7].median()
        out.append(float(np.float32(q.item())))
    return out


def _run(feed, det, ref, calls):
    """`calls` engine calls into the detector and the reference; -> the reference's events"""
    out = []
    for _ in range(calls):
        probs, pending = feed.call()
        assert pending == det.pending_rows
        det.update(probs)
        out.append(ref.update([p.cpu().numpy() for p in probs], [p.shape[1] for p in probs], pending))
    return np.concatenate(out)


def _ref(feed, cutoffs, roles=(WAKE, WAKE, VAD)):
    e = feed.eng
    return ModelsRef(e.n_streams, list(roles), [WIN_WAKE, WIN_WAKE, WIN_VAD], cutoffs, [COOLDOWN] * 3, e.stride, e.streams)


def _drain_all(det):
    ev, dropped = det.drain()
    assert dropped == 0
    return ev


@pytest.mark.parametrize("S,sets", [(4096, False), (4096, True), (65536, True)])
def test_events_and_state_equal_the_reference(torch_cuda, S, sets):
    torch = torch_cuda
    from microwakeword_b200.detection import MultiModelDetector
    feed = Feed(torch, S, _sets(S, sets), seed=11 + S)
    assert feed.eng.stride == [3, 3, 17]
    cutoffs = _cutoffs(torch, feed)
    # created mid-stream: the models hold pending rows that differ
    det = MultiModelDetector(feed.eng, cutoffs, [WIN_WAKE, WIN_WAKE, WIN_VAD], COOLDOWN, vad=2, capacity=1 << 20)
    ref = _ref(feed, cutoffs)
    ungated = _ref(feed, cutoffs, (WAKE, WAKE, OFF))
    calls = 300 if S <= 4096 else 120
    got, want, free = [], [], []
    for c in range(calls):
        probs, pending = feed.call()
        det.update(probs)
        host = [p.cpu().numpy() for p in probs]
        n = [p.shape[1] for p in probs]
        want.append(ref.update(host, n, pending))
        free.append(ungated.update(host, n, pending))
        if c % 97 == 50:
            got.append(_drain_all(det))
    got.append(_drain_all(det))
    got, want, free = (np.concatenate(x) for x in (got, want, free))
    assert same_model_events(got, want)
    assert same_model_state(det.state_dict()["models"], ref.state())
    assert det.pending_rows == feed.eng.pending_rows
    # both wake words fired, on streams of their sets only, and the VAD refused some candidates
    for k in (0, 1):
        mine = got[got["model"] == k]
        assert mine.size > 0 and np.isin(mine["stream"], feed.eng.streams[k]).all()
    assert want.size < free.size


def test_without_a_vad_each_model_is_a_stream_detector(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    S = 4096
    feed = Feed(torch, S, _sets(S, True, seed=5), seed=21)
    cutoffs = _cutoffs(torch, feed)
    det = MultiModelDetector(feed.eng, cutoffs, [WIN_WAKE, WIN_WAKE, WIN_VAD], COOLDOWN)
    plain = [StreamDetector(feed.eng.streams[k].size, cutoffs[k], w, COOLDOWN, stream_ids=feed.eng.streams[k])
             for k, w in enumerate((WIN_WAKE, WIN_WAKE, WIN_VAD))]
    for _ in range(150):
        probs, _ = feed.call()
        det.update(probs)
        for d, p in zip(plain, probs):
            d.update(p)
    got = _drain_all(det)
    for k in range(3):
        want = _drain_all(plain[k])
        assert want.size > 0 and same_events(got[got["model"] == k], want), k
        s = det.state_dict()["models"][k]
        assert same_state(s, plain[k].state_dict())


def test_fired_ids_restart_exactly_those_streams_and_state_moves(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import MultiModelDetector
    S = 4096
    feed = Feed(torch, S, None, seed=31)
    twin = Feed(torch, S, None, seed=31)
    cutoffs = _cutoffs(torch, feed)
    _cutoffs(torch, twin)
    det = MultiModelDetector(feed.eng, cutoffs, [WIN_WAKE, WIN_WAKE, WIN_VAD], COOLDOWN, vad=2)
    ref = _ref(feed, cutoffs)
    for _ in range(80):
        probs, pending = feed.call()
        twin.call()
        det.update(probs)
        ref.update([p.cpu().numpy() for p in probs], [p.shape[1] for p in probs], pending)
    fired_list = det.fired_ids.cpu().numpy()
    fired = np.unique(fired_list[fired_list >= 0])
    assert 0 < fired.size < S
    before = feed.eng.state_dict()
    feed.eng.reset(det.fired_ids)                            # no host round trip: the list the kernel wrote
    det.reset(det.fired_ids)
    ev = _drain_all(det)
    assert np.array_equal(np.unique(ev["stream"]), fired) and (det.fired_ids.cpu().numpy() == -1).all()
    ref.reset(fired)
    twin.eng.reset(fired.tolist())
    after = feed.eng.state_dict()
    assert np.array_equal(after["carry"], twin.eng.state_dict()["carry"])
    others = np.setdiff1d(np.arange(S), fired)
    assert np.array_equal(after["carry"][others], before["carry"][others])
    assert same_model_state(det.state_dict()["models"], ref.state())
    # the state moves to a second detector of the same engine, which continues exactly as the first
    second = MultiModelDetector(feed.eng, cutoffs, [WIN_WAKE, WIN_WAKE, WIN_VAD], COOLDOWN, vad=2)
    second.load_state_dict(det.state_dict())
    want = []
    for _ in range(60):
        probs, pending = feed.call()
        det.update(probs)
        second.update(probs)
        want.append(ref.update([p.cpu().numpy() for p in probs], [p.shape[1] for p in probs], pending))
    want = np.concatenate(want)
    assert want.size > 0
    for d in (det, second):
        assert same_model_events(_drain_all(d), want)
        assert same_model_state(d.state_dict()["models"], ref.state())
    # a full reset after engine.reset() starts every stream over and re-reads the pending rows
    feed.eng.reset()
    det.reset()
    assert det.pending_rows == feed.eng.pending_rows == [0, 0, 0]
    fresh = _ref(feed, cutoffs)
    want = _run(feed, det, fresh, 40)
    assert same_model_events(_drain_all(det), want)
    assert same_model_state(det.state_dict()["models"], fresh.state())


def test_refusals_leave_the_state_unchanged(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    S = 512
    feed = Feed(torch, S, _sets(S, True, seed=9), seed=41)
    cutoffs = _cutoffs(torch, feed, 20)
    det = MultiModelDetector(feed.eng, cutoffs, [WIN_WAKE, WIN_WAKE, WIN_VAD], COOLDOWN, vad=2)
    for _ in range(30):
        det.update(feed.call()[0])
    L = _lib.lib()
    state = det.state_dict()
    count = int(det.event_count.item())

    def unchanged():
        torch.cuda.synchronize()
        return same_model_state(det.state_dict()["models"], state["models"]) and int(det.event_count.item()) == count

    probs, pending = feed.call()
    K = 3
    steps = [p.shape[1] for p in probs]
    wide = [torch.zeros((p.shape[0], 8), device=p.device) for p in probs]     # room for every step count tried below
    ptrs = (ctypes.c_void_p * K)(*[w.data_ptr() for w in wide])
    pitch = (ctypes.c_longlong * K)(8, 8, 8)
    assert max(steps) > 0
    for n, p in (([steps[0] + 1, steps[1], steps[2]], pending), (steps, [pending[0], pending[1], 17]),
                 (steps, [pending[0], -1, pending[2]]), ([steps[0], steps[1], steps[2] + 2], pending)):
        rc = L.mww_multi_detector_update(det._d, ptrs, pitch, (ctypes.c_int * K)(*n), (ctypes.c_int * K)(*p), None)
        assert rc == -1 and b"one call" in L.mww_last_error(None), (n, p)
        assert unchanged()
    assert L.mww_multi_detector_update(det._d, ptrs, (ctypes.c_longlong * K)(0, 0, 0), (ctypes.c_int * K)(*steps),
                                        (ctypes.c_int * K)(*pending), None) == -1
    # wrong shapes, a stale stream set
    with pytest.raises(ValueError):
        det.update(probs[:2])
    with pytest.raises(ValueError):
        det.update([probs[0][:-1], probs[1], probs[2]])
    with pytest.raises(ValueError):
        det.update([probs[0].double(), probs[1], probs[2]])
    assert unchanged()
    # the plain calls on a models detector, and the reverse
    assert L.mww_detector_update(det._d, probs[0].data_ptr(), 1, 1, None) == -1
    assert L.mww_detector_get_state(det._d, None, None, None) == -1 and L.mww_detector_set_state(det._d, None, None, None) == -1
    plain = StreamDetector(8, 0.5)
    z = (ctypes.c_int * K)(0, 0, 0)
    assert L.mww_multi_detector_update(plain._d, ptrs, pitch, z, z, None) == -1
    assert L.mww_multi_detector_get_state(plain._d, 0, None, None, None) == -1
    # model state: out-of-range values and indices, checked before anything is written
    bad = det.state_dict()
    bad["models"][2]["active"][0] = 2
    with pytest.raises(ValueError):
        det.load_state_dict(bad)
    n0 = feed.eng.streams[0].size
    cd = np.full(n0, COOLDOWN + 1, np.int32)
    assert L.mww_multi_detector_set_state(det._d, 0, None, None, cd.ctypes.data) == -1
    seen = np.full(n0, -1, np.int64)
    assert L.mww_multi_detector_set_state(det._d, 0, None, seen.ctypes.data, None) == -1
    assert L.mww_multi_detector_get_state(det._d, 3, None, None, None) == -1
    assert unchanged()
    # creation: two VADs, no WAKE, a bad role or window; an OFF model has no state
    d = ctypes.c_void_p()
    for roles, window, word in (((VAD, WAKE, VAD), 5, b"VAD"), ((VAD, OFF, OFF), 5, b"WAKE"), ((WAKE, 7, OFF), 5, b"role"),
                                ((WAKE, WAKE, OFF), 33, b"window")):
        rules = (_lib.MwwDetectRule * K)(*[_lib.MwwDetectRule(r, window, 3, 0, 0.5) for r in roles])
        assert L.mww_multi_detector_create(feed.eng._h, rules, 16, ctypes.byref(d)) == -1 and word in L.mww_last_error(None)
        assert not d.value
    off = MultiModelDetector(feed.eng, [cutoffs[0], None, None], WIN_WAKE, COOLDOWN)
    assert L.mww_multi_detector_get_state(off._d, 1, None, None, None) == -1
    assert off.state_dict()["models"][1] is None
    off.update([feed.call()[0][0], None, None])               # an OFF model's entry is not read
    # a frontend-only handle
    from microwakeword_b200.engine import StreamEngine
    front = StreamEngine(None, 16)
    rules = (_lib.MwwDetectRule * 1)(_lib.MwwDetectRule(WAKE, 5, 3, 0, 0.5))
    assert L.mww_multi_detector_create(front._h, rules, 16, ctypes.byref(d)) == -1 and b"frontend-only" in L.mww_last_error(None)
    # after set_streams the detector's sets are stale
    feed.eng.set_streams(1, None)
    with pytest.raises(ValueError):
        det.update(feed.call()[0])
