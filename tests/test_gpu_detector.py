"""The streaming detector on the GPU (run with -m gpu on an H100): detector_update_kernel in both forms against the NumPy
reference (tests/detector_ref.py), events as sorted sets with scores bit for bit, at 65 509 rows (a short last warp and
block); overflow of the event buffer; row pitch, empty calls, the row -> stream map, resets by row, state moved between
detectors; and behind the real engines, where the fired-id list restarts the streams that fired."""

import os

import numpy as np
import pytest

from conftest import GOLDEN
from detector_ref import DetectorRef, same_events, same_state, sort_events

pytestmark = pytest.mark.gpu

R_FULL = 65509


def _detector(*a, **kw):
    from microwakeword_b200.detection import StreamDetector
    return StreamDetector(*a, **kw)


def _seeded_probs(rows, steps, seed, share=0.01):
    """background below the cutoff; `share` of the rows get a burst above it somewhere, a few stay high throughout"""
    rng = np.random.default_rng(seed)
    p = (rng.random((rows, steps)) * 0.4).astype(np.float32)
    hot = rng.choice(rows, max(int(rows * share), 4), replace=False)
    for r in hot:
        at = int(rng.integers(0, steps - 8))
        p[r, at:at + int(rng.integers(3, 12))] = np.float32(0.7 + 0.3 * rng.random())
    p[hot[:3]] = 0.97
    p[hot[3], steps // 2] = np.nan
    return p


def _drain_all(det):
    ev, dropped = det.drain()
    assert dropped == 0
    return ev


def test_live_and_clip_shapes_equal_the_reference_at_full_size(torch_cuda):
    torch = torch_cuda
    steps, cutoff, window, cooldown = 120, 0.6, 5, 25
    probs = _seeded_probs(R_FULL, steps, 1)
    ref = DetectorRef(R_FULL, cutoff, window, cooldown)
    want = ref.update(probs)
    fired_rows = np.unique(want["stream"]).size
    assert 0.003 * R_FULL < fired_rows < 0.02 * R_FULL and want.size > fired_rows
    dev = torch.from_numpy(probs).cuda()

    live = _detector(R_FULL, cutoff, window, cooldown)
    got, drains = [], {2, 16, 17, 59, 118}
    for t in range(steps):
        live.update(dev[:, t:t + 1])                       # a column of the wider buffer, read in place
        if t in drains:
            got.append(_drain_all(live))
    got.append(_drain_all(live))
    assert all((np.diff(g["step"]) >= 0).all() for g in got)
    assert same_events(np.concatenate(got), want)
    assert same_state(live.state_dict(), ref.state())

    one = _detector(R_FULL, cutoff, window, cooldown)
    one.update(dev)
    assert same_events(_drain_all(one), want) and same_state(one.state_dict(), ref.state())

    three = _detector(R_FULL, cutoff, window, cooldown)
    for a, b in ((0, 7), (7, 107), (107, 120)):            # thread form, warp form over several passes, warp form in one
        three.update(dev[:, a:b])
    assert same_events(_drain_all(three), want) and same_state(three.state_dict(), ref.state())


@pytest.mark.parametrize("window,cooldown", [(1, 0), (32, 3)])
def test_window_extremes(torch_cuda, window, cooldown):
    torch = torch_cuda
    rows, steps = 1000, 150
    probs = np.random.default_rng(window).random((rows, steps)).astype(np.float32)
    ref = DetectorRef(rows, 0.52, window, cooldown)
    want = ref.update(probs)
    assert want.size > rows
    dev = torch.from_numpy(probs).cuda()
    det = _detector(rows, 0.52, window, cooldown, capacity=want.size)
    for a, b in ((0, 3), (3, 4), (4, 70), (70, 71), (71, 150)):
        det.update(dev[:, a:b])
    assert same_events(_drain_all(det), want) and same_state(det.state_dict(), ref.state())


def test_overflow_counts_every_event_and_keeps_the_state(torch_cuda):
    torch = torch_cuda
    rows, steps, capacity = 4096, 40, 16
    probs = np.full((rows, steps), 0.9, np.float32)
    ref = DetectorRef(rows, 0.5, 5, 10)
    want = ref.update(probs)
    assert want.size > rows
    dev = torch.from_numpy(probs).cuda()
    det = _detector(rows, 0.5, 5, 10, capacity=capacity)
    assert (det.fired_ids.cpu().numpy() == -1).all()
    det.update(dev)
    fired = det.fired_ids.cpu().numpy()
    assert int(det.event_count.cpu()) == want.size and (fired >= 0).all()
    ev, dropped = det.drain()
    assert ev.size == capacity and dropped == want.size - capacity
    true = {(int(e["stream"]), int(e["step"]), np.float32(e["score"]).tobytes()) for e in want}
    assert len({(int(e["stream"]), int(e["step"])) for e in ev}) == capacity
    assert all((int(e["stream"]), int(e["step"]), np.float32(e["score"]).tobytes()) in true for e in ev)
    assert sorted(fired.tolist()) == sorted(ev["stream"].tolist())
    assert same_state(det.state_dict(), ref.state())
    assert (det.fired_ids.cpu().numpy() == -1).all() and int(det.event_count.cpu()) == 0
    ev, dropped = det.drain()
    assert ev.size == 0 and dropped == 0
    # live calls overflow the same way
    det.update(dev[:, :1])
    det.update(dev[:, 1:2])
    ev, dropped = det.drain()
    want2 = ref.update(probs[:, :2])
    assert ev.size + dropped == want2.size and same_state(det.state_dict(), ref.state())


def test_pitch_empty_calls_and_the_stream_map(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200 import _lib
    rows, steps = 777, 64
    probs = _seeded_probs(rows, steps, 2, share=0.1)
    ids = (np.arange(rows, dtype=np.int32) * 3 + 100)
    ref = DetectorRef(rows, 0.6, 5, 4, stream_ids=ids)
    want = ref.update(probs)
    assert want.size > 20
    wide = torch.full((rows, 200), 5.0, dtype=torch.float32, device="cuda")         # anything read past the steps would fire
    wide[:, :steps] = torch.from_numpy(probs).cuda()
    det = _detector(rows, 0.6, 5, 4, stream_ids=ids)
    before = det.state_dict()
    det.update(wide[:, :0])
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert _lib.lib().mww_detector_update(det._d, wide.data_ptr(), 0, 200, None) == 0
        torch.cuda.synchronize()
    assert not [e.key for e in prof.key_averages() if "detector" in e.key]
    assert same_state(det.state_dict(), before)
    det.update(wide[:, :5])
    det.update(wide[:, 5:steps])
    got = _drain_all(det)
    assert same_events(got, want) and set(got["stream"].tolist()) <= set(ids.tolist())
    assert _lib.lib().mww_detector_update(det._d, wide.data_ptr(), 8, 7, None) == -1        # a pitch below the steps
    with pytest.raises(ValueError):
        det.update(wide[:5, :4])
    with pytest.raises(ValueError):
        det.update(wide[:, :4].double())


def test_reset_by_row_from_host_and_device_lists(torch_cuda):
    torch = torch_cuda
    rows, cutoff, window, cooldown = 3001, 0.5, 5, 3
    rng = np.random.default_rng(4)
    probs = rng.random((rows, 40)).astype(np.float32)
    dev = torch.from_numpy(probs).cuda()
    for from_device in (False, True):
        ref = DetectorRef(rows, cutoff, window, cooldown)
        det = _detector(rows, cutoff, window, cooldown)
        det.update(dev[:, :20])
        want = [ref.update(probs[:, :20])]
        before = det.state_dict()
        listed = np.asarray([5, 2999, 5, -1, rows, 3000, 64, 2 ** 30], np.int32)          # twice, and out of range
        det.reset(torch.from_numpy(listed).cuda() if from_device else listed)
        ref.reset(listed)
        after = det.state_dict()
        assert same_state(after, ref.state())
        hit = np.zeros(rows, bool)
        hit[[5, 2999, 3000, 64]] = True
        assert (after["seen"][hit] == 0).all() and (after["cooldown"][hit] == cooldown).all() and not after["hist"][hit].any()
        for k in before:                                   # every other row's state bytes are unchanged
            assert np.array_equal(before[k][~hit].view(np.uint8), after[k][~hit].view(np.uint8))
        det.update(dev[:, 20:23])                          # reset rows warm up again: nothing from them for window - 1 steps
        ev = ref.update(probs[:, 20:23])
        assert not np.isin(ev["stream"], [5, 2999, 3000, 64]).any()
        want.append(ev)
        det.update(dev[:, 23:])
        want.append(ref.update(probs[:, 23:]))
        assert same_events(_drain_all(det), np.concatenate(want)) and same_state(det.state_dict(), ref.state())
        det.reset()
        ref.reset()
        assert same_state(det.state_dict(), ref.state())


def test_state_moves_to_a_second_detector_and_continues_bit_for_bit(torch_cuda):
    torch = torch_cuda
    rows = 513
    probs = np.random.default_rng(6).random((rows, 90)).astype(np.float32)
    dev = torch.from_numpy(probs).cuda()
    ref = DetectorRef(rows, 0.55, 7, 5)
    a = _detector(rows, 0.55, 7, 5)
    a.update(dev[:, :37])
    ref.update(probs[:, :37])
    _drain_all(a)
    b = _detector(rows, 0.55, 7, 5)
    b.load_state_dict(a.state_dict())
    assert same_state(b.state_dict(), a.state_dict())
    for d in (a, b):
        d.update(dev[:, 37:40])
        d.update(dev[:, 40:])
    want = sort_events(np.concatenate([ref.update(probs[:, 37:40]), ref.update(probs[:, 40:])]))
    ea, eb = _drain_all(a), _drain_all(b)
    assert same_events(ea, want) and same_events(eb, want)
    assert same_state(a.state_dict(), ref.state()) and same_state(b.state_dict(), ref.state())
    from microwakeword_b200 import _lib
    bad = a.state_dict()
    bad["cooldown"][3] = 6
    with pytest.raises(_lib.MwwError):
        b.load_state_dict(bad)
    with pytest.raises(ValueError):
        b.load_state_dict(dict(bad, seen=bad["seen"][:5]))


# ---- behind the engines ------------------------------------------------------------------------------------------------------
def _blob(kind):
    return open(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % kind), "rb").read()


def _audio():
    return np.load(os.path.join(GOLDEN, "batch_audio.npy"))


def _cutoff_in_a_gap(probs, window, cooldown):
    """a cutoff inside the observed range at which some streams fire and others do not, as far from every moving average
    as such a cutoff can be: a last-bit difference between two kernels cannot change a decision"""
    from oracle import detection_ref as D
    avg = np.stack([D.moving_average(t, window) for t in probs]).astype(np.float64)
    levels = np.unique(avg)
    best = (0.0, None)
    for m in (levels[1:] + levels[:-1]) / 2:
        m = float(np.float32(m))
        fired = np.unique(DetectorRef(len(probs), m, window, cooldown).update(probs)["stream"]).size
        if 0 < fired < len(probs):
            best = max(best, (float(np.abs(avg - m).min()), m))
    assert best[0] > 1e-4
    return best[1]


def _state_equal(a, b, rows=None):
    for k in ("carry", "estimate", "nn", "pending"):
        x, y = (a[k], b[k]) if rows is None else (a[k][rows], b[k][rows])
        if not np.array_equal(x.view(np.uint8), y.view(np.uint8)):
            return False
    return rows is not None or (a["frontend_buffered"], a["pending_rows"]) == (b["frontend_buffered"], b["pending_rows"])


@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_detections_of_a_live_engine_and_restart_of_the_streams_that_fired(torch_cuda, kind):
    torch = torch_cuda
    from microwakeword_b200.engine import StreamEngine
    audio = _audio()
    S, n_calls, window, cooldown = audio.shape[0], audio.shape[1] // 480, 5, 2
    dev = torch.from_numpy(audio).cuda()
    clip = StreamEngine(_blob(kind), S).predict_clip(dev[:, :480 * n_calls].contiguous()).cpu().numpy()
    cutoff = _cutoff_in_a_gap(clip, window, cooldown)

    eng, twin = StreamEngine(_blob(kind), S), StreamEngine(_blob(kind), S)
    det = _detector(S, cutoff, window, cooldown)
    live = []
    for i in range(n_calls):
        chunk = dev[:, 480 * i:480 * (i + 1)].contiguous()
        p = eng.step(chunk)
        twin.step(chunk)
        det.update(p)                                      # the sliced result of step(), as it is
        live.append(p.cpu().numpy())
    live = np.concatenate(live, 1)
    assert live.shape == clip.shape
    fired_list = det.fired_ids.cpu().numpy()
    before = eng.state_dict()
    eng.reset(det.fired_ids)                               # no host round trip: the list the kernels wrote
    got = _drain_all(det)
    # the reference on exactly the probabilities the detector consumed: bit for bit
    assert same_events(got, DetectorRef(S, cutoff, window, cooldown).update(live))
    # and on predict_clip's probabilities for the same audio
    want = DetectorRef(S, cutoff, window, cooldown).update(clip)
    fired = np.unique(want["stream"])
    assert 0 < fired.size < S
    assert np.array_equal(got["stream"], want["stream"]) and np.array_equal(got["step"], want["step"])
    if kind == "int8":
        assert same_events(got, want)
    else:
        assert np.abs(got["score"] - want["score"]).max() <= 1e-5
    assert np.array_equal(np.unique(fired_list[fired_list >= 0]), fired)
    assert (det.fired_ids.cpu().numpy() == -1).all()
    # the fired streams are in the state mww_reset(ids) gives, the others untouched
    twin.reset(fired.tolist())
    after = eng.state_dict()
    assert _state_equal(after, twin.state_dict())
    others = np.setdiff1d(np.arange(S), fired)
    assert _state_equal(after, before, others) and not _state_equal(after, before, fired)


def test_one_detector_per_model_of_a_handle_with_stream_sets(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.engine import MultiModelEngine
    audio = _audio()
    S, n_calls, window, cooldown = audio.shape[0], audio.shape[1] // 480, 5, 2
    dev = torch.from_numpy(audio).cuda()
    sets = [None, [1, 4, 5, 9, 11]]
    blobs = [_blob("f32"), _blob("int8")]
    clip = [p.cpu().numpy() for p in MultiModelEngine(blobs, S, streams=sets).predict_clip(dev[:, :480 * n_calls].contiguous())]
    eng = MultiModelEngine(blobs, S, streams=sets)
    assert eng.streams[1].tolist() == sets[1]
    cutoffs = [_cutoff_in_a_gap(c, window, cooldown) for c in clip]
    dets = [_detector(eng.streams[k].size, cutoffs[k], window, cooldown, stream_ids=eng.streams[k]) for k in range(2)]
    live = [[], []]
    for i in range(n_calls):
        for k, p in enumerate(eng.step(dev[:, 480 * i:480 * (i + 1)].contiguous())):
            dets[k].update(p)
            live[k].append(p.cpu().numpy())
    for k in range(2):
        got = _drain_all(dets[k])
        ref = DetectorRef(eng.streams[k].size, cutoffs[k], window, cooldown, stream_ids=eng.streams[k])
        assert same_events(got, ref.update(np.concatenate(live[k], 1)))
        want = DetectorRef(eng.streams[k].size, cutoffs[k], window, cooldown, stream_ids=eng.streams[k]).update(clip[k])
        assert want.size > 0 and np.array_equal(got["stream"], want["stream"]) and np.array_equal(got["step"], want["step"])
        assert set(got["stream"].tolist()) <= set(eng.streams[k].tolist())
