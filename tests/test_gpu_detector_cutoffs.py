"""Per-row cutoffs on the GPU (run with -m gpu on an H100): StreamDetector and MultiModelDetector after set_cutoffs, against
the NumPy reference (tests/detector_cutoffs_ref.py) and against uniform detectors, events as sets with scores bit for bit and
the final state bit for bit.  65 509 rows in live, clip and mixed calls; all-equal cutoffs against uniform mode; cutoff
changes mid-run; fired-id restarts behind a StreamEngine; the models detector behind a MultiModelEngine at 65 536 streams with
and without stream sets, on the engine's own probabilities; refusals that leave state and cutoffs unchanged."""

import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from detector_cutoffs_ref import ModelsRowsRef, RowsRef
from detector_models_ref import VAD, WAKE, same_model_events, same_model_state
from detector_ref import same_events, same_state

pytestmark = pytest.mark.gpu

R_FULL = 65509
LEVELS = (0.55, 0.7, 0.85)


def _drain_all(det):
    ev, dropped = det.drain()
    assert dropped == 0
    return ev


def _probs(rows, steps, seed):
    """background below the levels, bursts in a few percent of the rows, a NaN"""
    rng = np.random.default_rng(seed)
    p = (rng.random((rows, steps)) * 0.5).astype(np.float32)
    hot = rng.choice(rows, rows // 20, replace=False)
    for r in hot:
        at = int(rng.integers(0, steps - 8))
        p[r, at:at + int(rng.integers(3, 12))] = np.float32(0.5 + 0.5 * rng.random())
    p[hot[0], steps // 2] = np.nan
    return p


def _levels(rows, seed):
    """(per-row cutoffs, level index per row, -1 for a random cutoff)"""
    rng = np.random.default_rng(seed)
    level = rng.integers(0, 3, rows)
    level[rng.random(rows) < 0.1] = -1
    c = np.where(level >= 0, np.asarray(LEVELS)[np.maximum(level, 0)], rng.uniform(0.5, 0.95, rows))
    return c, level


def _state_rows(state, rows):
    return {k: v[rows] for k, v in state.items()}


def test_plain_detector_at_full_size_in_three_call_shapes(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import StreamDetector
    steps, window, cooldown = 120, 5, 25
    probs = _probs(R_FULL, steps, 1)
    cut, level = _levels(R_FULL, 2)
    ref = RowsRef(R_FULL, LEVELS[1], window, cooldown)
    ref.set_cutoffs(np.arange(R_FULL), cut)
    want = ref.update(probs)
    assert all((want["stream"][np.isin(want["stream"], np.flatnonzero(level == L))]).size > 0 for L in range(3))
    dev = torch.from_numpy(probs).cuda()
    shapes = {"live": [(t, t + 1) for t in range(steps)], "clip": [(0, steps)], "mixed": [(0, 7), (7, 107), (107, 120)]}
    for name, calls in shapes.items():
        det = StreamDetector(R_FULL, LEVELS[1], window, cooldown, capacity=1 << 20)
        det.set_cutoffs(np.arange(R_FULL), cut)
        assert np.array_equal(det.cutoffs, cut)
        for a, b in calls:
            det.update(dev[:, a:b])
        got = _drain_all(det)
        assert same_events(got, want), name
        assert same_state(det.state_dict(), ref.state()), name
    # (b) a uniform detector at each level, restricted to that level's rows
    for L, c in enumerate(LEVELS):
        uni = StreamDetector(R_FULL, c, window, cooldown, capacity=1 << 20)
        uni.update(dev)
        u = _drain_all(uni)
        rows = np.flatnonzero(level == L)
        assert same_events(u[np.isin(u["stream"], rows)], got[np.isin(got["stream"], rows)]), c
        assert same_state(_state_rows(uni.state_dict(), rows), _state_rows(det.state_dict(), rows))


def test_all_equal_cutoffs_are_uniform_mode_and_changes_mid_run(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import StreamDetector
    R, steps, window, cooldown = 4099, 90, 5, 10
    probs = _probs(R, steps, 3)
    dev = torch.from_numpy(probs).cuda()
    uni = StreamDetector(R, 0.6, window, cooldown)
    per = StreamDetector(R, 0.6, window, cooldown)
    assert np.array_equal(per.cutoffs, np.full(R, 0.6))
    per.set_cutoffs([], [])                                 # n == 0: nothing, and still uniform mode
    per.set_cutoffs(np.arange(R), 0.6)
    for a, b in ((0, 1), (1, 50), (50, 51), (51, 90)):
        uni.update(dev[:, a:b])
        per.update(dev[:, a:b])
    assert same_events(_drain_all(per), _drain_all(uni)) and same_state(per.state_dict(), uni.state_dict())

    # changes between calls, resets in between (which keep the cutoffs), against the reference
    cut, _ = _levels(R, 4)
    det = StreamDetector(R, 0.6, window, cooldown)
    ref = RowsRef(R, 0.6, window, cooldown)
    rng = np.random.default_rng(5)
    got, want = [], []
    for i, (a, b) in enumerate(((0, 3), (3, 60), (60, 61), (61, 62), (62, 90))):
        rows = rng.choice(R, 300, replace=False) if i else np.arange(R)
        vals = cut[rows] if i == 0 else rng.uniform(0.4, 0.9, rows.size)
        for d in (det, ref):
            d.set_cutoffs(rows, vals)
        if i == 3:
            for d in (det, ref):
                d.reset([0, 1, 2, 17, R + 5])
        det.update(dev[:, a:b])
        want.append(ref.update(probs[:, a:b]))
        got.append(_drain_all(det))
    assert same_events(np.concatenate(got), np.concatenate(want))
    assert same_state(det.state_dict(), ref.state()) and np.array_equal(det.cutoffs, ref.cutoffs())


def test_refusals_leave_state_and_cutoffs_unchanged(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    from microwakeword_b200.engine import MultiModelEngine
    R = 64
    det = StreamDetector(R, 0.5, 5, 3)
    det.update(torch.from_numpy(_probs(R, 20, 6)).cuda())
    before, cut0 = det.state_dict(), det.cutoffs
    L = _lib.lib()

    def call(rows, cuts, n=None):
        r, c = np.ascontiguousarray(rows, np.int32), np.ascontiguousarray(cuts, np.float64)
        return L.mww_set_detector_cutoffs(det._d, r.ctypes.data, c.ctypes.data, r.size if n is None else n, None), L.mww_last_error(None)

    for rows, cuts, n, word in (([1], [np.nan], None, b"finite"), ([1], [np.inf], None, b"finite"), ([R], [0.5], None, b"range"),
                                ([-1], [0.5], None, b"range"), ([3, 3], [0.5, 0.6], None, b"twice"), ([1], [0.5], -1, b"negative")):
        rc, msg = call(rows, cuts, n)
        assert rc == -1 and word in msg, (rows, msg)
    assert L.mww_set_detector_cutoffs(det._d, None, None, 1, None) == -1
    assert same_state(det.state_dict(), before) and np.array_equal(det.cutoffs, cut0)
    with pytest.raises(ValueError):
        det.set_cutoffs([1, 2], [0.5, np.nan])
    with pytest.raises(_lib.MwwError):
        det.set_cutoffs([1, 1], 0.5)
    det.set_cutoffs([5], 0.75)
    want = cut0.copy()
    want[5] = 0.75
    with pytest.raises(_lib.MwwError):
        det.set_cutoffs([2, R + 1], [0.1, 0.2])               # refused as a whole: row 2 keeps its cutoff
    assert np.array_equal(det.cutoffs, want) and same_state(det.state_dict(), before)

    S = 96
    blob = open(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"), "rb").read()
    eng = MultiModelEngine([blob, blob, blob], S, streams=[None, np.arange(10, 60, dtype=np.int32), None])
    md = MultiModelDetector(eng, [0.6, 0.6, None], 5, 3)
    ids, c = np.asarray([3], np.int32), np.asarray([0.5])
    # a plain call on a models detector and the reverse; an OFF model; a bad k; a non-member; a duplicate; a non-finite value
    assert L.mww_set_detector_cutoffs(md._d, ids.ctypes.data, c.ctypes.data, 1, None) == -1
    assert L.mww_get_detector_cutoffs(md._d, c.ctypes.data) == -1
    assert L.mww_set_multi_detector_cutoffs(det._d, 0, ids.ctypes.data, c.ctypes.data, 1, None) == -1
    assert L.mww_get_multi_detector_cutoffs(det._d, 0, c.ctypes.data) == -1
    for k, sid, v, word in ((2, [3], [0.5], b"OFF"), (3, [3], [0.5], b"range"), (-1, [3], [0.5], b"range"), (1, [3], [0.5], b"member"),
                            (1, [12, 12], [0.5, 0.5], b"twice"), (0, [S], [0.5], b"range"), (0, [4], [np.nan], b"finite")):
        a, b = np.asarray(sid, np.int32), np.asarray(v, np.float64)
        assert L.mww_set_multi_detector_cutoffs(md._d, k, a.ctypes.data, b.ctypes.data, a.size, None) == -1, (k, sid)
        assert word in L.mww_last_error(None), (k, L.mww_last_error(None))
    assert L.mww_set_multi_detector_cutoffs(md._d, 0, ids.ctypes.data, c.ctypes.data, -1, None) == -1
    assert np.array_equal(md.get_cutoffs(0), np.full(S, 0.6)) and np.array_equal(md.get_cutoffs(1), np.full(50, 0.6))
    with pytest.raises(ValueError):
        md.set_cutoffs(2, [3], 0.5)
    md.set_cutoffs(1, [10, 59], [0.2, 0.3])
    got = md.get_cutoffs(1)
    assert got[0] == 0.2 and got[-1] == 0.3 and (got[1:-1] == 0.6).all() and np.array_equal(md.get_cutoffs(0), np.full(S, 0.6))


def test_fired_ids_restart_the_streams_behind_a_stream_engine(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import StreamDetector
    from microwakeword_b200.engine import StreamEngine
    audio = np.load(os.path.join(GOLDEN, "batch_audio.npy"))
    S, n_calls = audio.shape[0], audio.shape[1] // 480
    blob = open(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"), "rb").read()
    dev = torch.from_numpy(audio).cuda()
    eng, twin = StreamEngine(blob, S), StreamEngine(blob, S)
    live = []
    for i in range(n_calls):
        chunk = dev[:, 480 * i:480 * (i + 1)].contiguous()
        live.append(twin.step(chunk).cpu().numpy())
    live = np.concatenate(live, 1)
    # per-row cutoffs just below or above each stream's best average after the first (the initial cooldown of 2 steps keeps
    # the first average from firing): about half the streams fire
    avg = np.stack([np.convolve(t, np.ones(5) / 5, "valid") for t in live.astype(np.float64)])[:, 1:]
    rng = np.random.default_rng(8)
    cut = np.where(rng.random(S) < 0.5, avg.max(1) - 1e-4, avg.max(1) + 1e-3)
    det = StreamDetector(S, 0.5, 5, 2)
    det.set_cutoffs(np.arange(S), cut)
    for i in range(n_calls):
        det.update(eng.step(dev[:, 480 * i:480 * (i + 1)].contiguous()))
    fired_list = det.fired_ids.cpu().numpy()
    eng.reset(det.fired_ids)
    ref = RowsRef(S, 0.5, 5, 2)
    ref.set_cutoffs(np.arange(S), cut)
    want = ref.update(live)
    got = _drain_all(det)
    assert same_events(got, want)
    fired = np.unique(want["stream"])
    assert 0 < fired.size < S and np.array_equal(np.unique(fired_list[fired_list >= 0]), fired)
    twin.reset(fired.tolist())
    a, b = eng.state_dict(), twin.state_dict()
    assert all(np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)) for k in ("carry", "estimate", "nn", "pending"))


# ---- the models detector behind a MultiModelEngine ------------------------------------------------------------------------------
def _engine(S, sets):
    from microwakeword_b200.engine import MultiModelEngine
    f32, i8 = (open(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % k), "rb").read() for k in ("f32", "int8"))
    streams = None
    if sets:
        rng = np.random.default_rng(3)
        streams = [None, np.flatnonzero(rng.random(S) < 0.6).astype(np.int32), np.flatnonzero(rng.random(S) < 0.7).astype(np.int32)]
    return MultiModelEngine([f32, i8, f32], S, streams=streams)


def _calls(torch, S, seed):
    sys.path.insert(0, ROOT)
    from bench import synth_audio_device
    dev = torch.device("cuda", 0)
    pool = [synth_audio_device(torch, S, 4800, seed + i, dev) for i in range(3)]
    rng = np.random.default_rng(seed)
    i = 0
    while True:
        n = 480 if rng.random() < 0.75 else int(rng.choice([800, 1440, 4800]))
        yield pool[i % 3][:, :n]
        i += 1


def _warm_cutoffs(torch, eng, calls, windows):
    """model cutoffs from 30 calls' probabilities: wake at the 80th percentile of the streams' best averages, VAD at the median"""
    got = [[], [], []]
    for _ in range(30):
        a = next(calls)
        for k, p in enumerate(eng.step(a) if a.shape[1] == 480 else eng.predict_clip(a)):
            got[k].append(p)
    out = []
    for k in range(3):
        avg = torch.cat(got[k], 1).unfold(1, windows[k], 1).mean(-1)
        q = avg.max(1).values.quantile(0.8) if k < 2 else avg.flatten()[::7].median()
        out.append(float(np.float32(q.item())))
    return out


@pytest.mark.parametrize("sets", [False, True])
def test_models_detector_with_per_stream_cutoffs_equals_the_reference(torch_cuda, sets):
    torch = torch_cuda
    from microwakeword_b200.detection import MultiModelDetector
    S, windows, cooldown = 65536, [5, 5, 3], 10
    eng = _engine(S, sets)
    calls = _calls(torch, S, 40 + sets)
    cut = _warm_cutoffs(torch, eng, calls, windows)
    det = MultiModelDetector(eng, cut, windows, cooldown, vad=2, capacity=1 << 20)
    ref = ModelsRowsRef(S, [WAKE, WAKE, VAD], windows, cut, [cooldown] * 3, eng.stride, eng.streams)
    rng = np.random.default_rng(9)
    for k in range(3):
        ids = eng.streams[k]
        vals = cut[k] + rng.choice([-0.02, 0.0, 0.02, 0.05], ids.size)
        det.set_cutoffs(k, ids, vals)
        ref.set_cutoffs(k, ids, vals)
    got, want = [], []
    for c in range(100):
        if c == 50:                                          # a change mid-run on every model
            for k in range(3):
                ids = eng.streams[k][::13]
                det.set_cutoffs(k, ids, 0.99 if k < 2 else 0.01)
                ref.set_cutoffs(k, ids, 0.99 if k < 2 else 0.01)
        a = next(calls)
        pending = eng.pending_rows
        probs = eng.step(a) if a.shape[1] == 480 else eng.predict_clip(a)
        det.update(probs)
        want.append(ref.update([p.cpu().numpy() for p in probs], [p.shape[1] for p in probs], pending))
        if c % 37 == 20:
            got.append(_drain_all(det))
    got.append(_drain_all(det))
    got, want = np.concatenate(got), np.concatenate(want)
    assert (got["model"] == 0).any() and (got["model"] == 1).any()
    assert same_model_events(got, want)
    assert same_model_state(det.state_dict()["models"], ref.state())
    assert all(np.array_equal(det.get_cutoffs(k), ref.get_cutoffs(k)) for k in range(3))


def test_models_detector_without_a_vad_is_per_row_stream_detectors(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    S, windows, cooldown = 65536, [5, 5, 3], 10
    eng = _engine(S, True)
    calls = _calls(torch, S, 60)
    cut = _warm_cutoffs(torch, eng, calls, windows)
    det = MultiModelDetector(eng, cut, windows, cooldown, capacity=1 << 20)
    plain = [StreamDetector(eng.streams[k].size, cut[k], windows[k], cooldown, capacity=1 << 20, stream_ids=eng.streams[k]) for k in range(3)]
    rng = np.random.default_rng(10)
    for k in range(3):
        vals = cut[k] + rng.uniform(-0.05, 0.05, eng.streams[k].size)
        det.set_cutoffs(k, eng.streams[k], vals)
        plain[k].set_cutoffs(np.arange(eng.streams[k].size), vals)
    for _ in range(80):
        a = next(calls)
        probs = eng.step(a) if a.shape[1] == 480 else eng.predict_clip(a)
        det.update(probs)
        for d, p in zip(plain, probs):
            d.update(p)
    got = _drain_all(det)
    state = det.state_dict()["models"]
    for k in range(3):
        mine = got[got["model"] == k]
        assert mine.size > 0
        assert same_events(mine, _drain_all(plain[k]))
        assert same_state(state[k], plain[k].state_dict())
