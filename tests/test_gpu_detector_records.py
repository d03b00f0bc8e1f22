"""Detector records on the GPU (run with -m gpu on an H100): rows moved with export_rows / import_rows and export_streams /
import_streams continue bit for bit as rows that never moved.  A 65 536-row StreamDetector grown into a 98 304-row one
through 100 live calls and a 150-step clip call (both kernel forms), with per-row cutoffs and rows in cooldown; a
WAKE + WAKE + VAD MultiModelDetector carried across engine.set_streams into a new detector (stayers continue, joiners start
fresh, the VAD gate carries over); a save / load checkpoint; refusals that change nothing; a launch count independent of n;
event buffers left alone."""

import ctypes

import numpy as np
import pytest

from conftest import GOLDEN  # noqa: F401
from detector_ref import same_events, same_state

pytestmark = pytest.mark.gpu

R_SRC, R_DST = 65536, 98304
WINDOW, COOLDOWN, BASE = 5, 25, 0.7


def _drain_all(det):
    ev, dropped = det.drain()
    assert dropped == 0
    return ev


def _probs(rows, steps, seed):
    """background below the cutoffs, bursts in a few percent of the rows (firing, then in cooldown), a NaN"""
    rng = np.random.default_rng(seed)
    p = (rng.random((rows, steps)) * 0.5).astype(np.float32)
    hot = rng.choice(rows, rows // 16, replace=False)
    for r in hot:
        at = int(rng.integers(0, steps - 8))
        p[r, at:at + int(rng.integers(3, 12))] = np.float32(0.75 + 0.25 * rng.random())
    p[hot[0], steps // 2] = np.nan
    return p


def _remap(ev, perm):
    ev = ev.copy()
    ev["stream"] = perm[ev["stream"]]
    return ev


def _rows(state, rows):
    return {k: v[rows] for k, v in state.items()}


# ---- growing a plain detector --------------------------------------------------------------------------------------------------
def test_growing_a_plain_detector_continues_bit_for_bit(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import StreamDetector
    rng = np.random.default_rng(1)
    src = StreamDetector(R_SRC, BASE, WINDOW, COOLDOWN, capacity=1 << 20)
    twin = StreamDetector(R_SRC, BASE, WINDOW, COOLDOWN, capacity=1 << 20)
    dst = StreamDetector(R_DST, BASE, WINDOW, COOLDOWN, capacity=1 << 20)
    cut_rows = rng.choice(R_SRC, R_SRC // 8, replace=False).astype(np.int32)
    cut = np.round(rng.uniform(0.55, 0.95, cut_rows.size), 3)
    for d in (src, twin):
        d.set_cutoffs(cut_rows, cut)
    warm = torch.from_numpy(_probs(R_SRC, 60, 2)).cuda()
    for t in range(60):                                     # live calls: firing rows, some still in cooldown at the move
        src.update(warm[:, t:t + 1])
        twin.update(warm[:, t:t + 1])
    assert same_events(_drain_all(src), _drain_all(twin))
    st = twin.state_dict()
    assert (st["cooldown"] > 0).sum() > 100 and (st["seen"] == 60).all()
    dst.update(torch.from_numpy(_probs(R_DST, 30, 3)).cuda())      # the destination's own rows hold state of their own
    _drain_all(dst)
    before = dst.state_dict()
    perm = rng.permutation(R_DST)[:R_SRC].astype(np.int32)        # row r of src -> row perm[r] of dst
    rec = src.export_rows(np.arange(R_SRC))
    assert rec.data.shape == (R_SRC, 48) and rec.layout.record_bytes == 48
    dst.import_rows(perm, rec)
    assert same_state(src.state_dict(), st)                      # export changed nothing
    after = dst.state_dict()
    assert same_state(_rows(after, perm), st)
    rest = np.setdiff1d(np.arange(R_DST), perm)
    assert same_state(_rows(after, rest), _rows(before, rest))   # unlisted rows keep their bytes
    assert np.array_equal(dst.cutoffs[perm], twin.cutoffs) and (dst.cutoffs[rest] == BASE).all()
    # 100 live calls (thread form), then one 150-step clip call (warp form)
    cont = _probs(R_SRC, 250, 4)
    big = _probs(R_DST, 250, 5)
    big[perm] = cont
    cont_d, big_d = torch.from_numpy(cont).cuda(), torch.from_numpy(big).cuda()
    for a, b in [(t, t + 1) for t in range(100)] + [(100, 250)]:
        twin.update(cont_d[:, a:b])
        dst.update(big_d[:, a:b])
    want = _remap(_drain_all(twin), perm)
    got = _drain_all(dst)
    assert want.size > 100
    assert same_events(got[np.isin(got["stream"], perm)], want)
    assert same_state(_rows(dst.state_dict(), perm), twin.state_dict())


# ---- changing a stream set -----------------------------------------------------------------------------------------------------
def _models_engine(S, sets):
    from bench import model_blob
    from microwakeword_b200.engine import MultiModelEngine
    return MultiModelEngine([model_blob("f32"), model_blob("int8"), model_blob("f32")], S, streams=sets)


RULES = dict(cutoffs=[0.7, 0.75, 0.5], windows=[5, 3, 10], cooldown_slices=[20, 10, 0], vad=2)


def _feed(torch, det, P, a, b):
    """steps [a, b) of the global probabilities P[k] [S, T] for det's members, one update"""
    det.update([torch.from_numpy(np.ascontiguousarray(P[k][det.streams[k], a:b])).cuda() for k in range(3)])


def test_changing_a_stream_set_keeps_the_stayers_rows(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import MultiModelDetector
    S, T = 8192, 200
    rng = np.random.default_rng(7)
    old_sets = [None, np.flatnonzero(rng.random(S) < 0.6).astype(np.int32), np.flatnonzero(rng.random(S) < 0.9).astype(np.int32)]
    eng, eng_twin = _models_engine(S, old_sets), _models_engine(S, old_sets)
    assert eng.stride == [3, 3, 3] and eng.pending_rows == [0, 0, 0]
    old = MultiModelDetector(eng, **RULES)
    twin = MultiModelDetector(eng_twin, **RULES)
    P = [_probs(S, T, 10), _probs(S, T, 11), np.full((S, T), 0.9, np.float32)]
    P[2][rng.random(S) < 0.2] = 0.1                                  # a fifth of the streams never speak
    # bursts right after the move, which only a carried VAD flag lets fire within the VAD's first window
    P[0][:S // 4, 60:66] = 0.95
    P[1][:S // 4, 60:64] = 0.95
    for d in (old, twin):
        d.set_cutoffs(0, np.arange(0, S, 5), 0.8)
        d.set_cutoffs(2, d.streams[2][::7], 0.4)
    for d in (old, twin):
        for t in range(30):
            _feed(torch, d, P, t, t + 1)
        _feed(torch, d, P, 30, 60)
    assert same_events(_drain_all(old), _drain_all(twin))
    # model 1 swaps a third of its set, the VAD drops a few streams and gains a few
    new1 = np.sort(np.concatenate([old_sets[1][::3], np.setdiff1d(np.arange(S), old_sets[1])[::2]])).astype(np.int32)
    new2 = np.sort(np.concatenate([old_sets[2][old_sets[2] % 50 != 0], np.setdiff1d(np.arange(S), old_sets[2])[::3]])).astype(np.int32)
    eng.set_streams(1, new1)
    eng.set_streams(2, new2)
    new = MultiModelDetector(eng, **RULES)
    ids = np.arange(S, dtype=np.int32)
    new.import_streams(ids, old.export_streams(ids))
    tw = twin.state_dict()["models"]
    got = new.state_dict()["models"]
    for k in range(3):
        o, n = twin.streams[k], new.streams[k]
        stay, join = np.intersect1d(o, n), np.setdiff1d(n, o)
        ro, rn = np.searchsorted(o, stay), np.searchsorted(n, stay)
        flag = "active" if k == 2 else "cooldown"
        assert all(np.array_equal(got[k][f][rn], tw[k][f][ro]) for f in ("hist", "seen", flag))
        rj = np.searchsorted(n, join)
        if k:
            assert join.size > 0
        assert not got[k]["hist"][rj].any() and not got[k]["seen"][rj].any()
        assert (got[k][flag][rj] == (0 if k == 2 else RULES["cooldown_slices"][k])).all()
        # cutoffs followed the stayers; joiners keep the model's
        assert np.array_equal(new.get_cutoffs(k)[rn], twin.get_cutoffs(k)[ro])
        assert (new.get_cutoffs(k)[rj] == RULES["cutoffs"][k]).all()
    assert (got[2]["active"] == 1).sum() > S // 2
    # stayers continue as the twin: first within the VAD's first window (gate carried), then the rest
    vad_same = np.isin(np.arange(S), old_sets[2]) == np.isin(np.arange(S), new2)
    for a, b in ((60, 66), (66, T)):
        for d in (new, twin):
            _feed(torch, d, P, a, b)
        g, w = _drain_all(new), _drain_all(twin)
        for k in range(2):
            stay = np.intersect1d(twin.streams[k], new.streams[k])
            stay = stay[vad_same[stay]]
            gk, wk = g[(g["model"] == k) & np.isin(g["stream"], stay)], w[(w["model"] == k) & np.isin(w["stream"], stay)]
            assert same_events(gk, wk), (a, k)
            if a == 60:
                assert wk.size > 50, k
    tw, got = twin.state_dict()["models"], new.state_dict()["models"]
    stay = np.intersect1d(twin.streams[2], new.streams[2])
    ro, rn = np.searchsorted(twin.streams[2], stay), np.searchsorted(new.streams[2], stay)
    assert all(np.array_equal(got[2][f][rn], tw[2][f][ro]) for f in ("hist", "seen", "active"))


# ---- checkpoint ---------------------------------------------------------------------------------------------------------------------
def test_checkpoint_save_and_load(torch_cuda, tmp_path):
    torch = torch_cuda
    from microwakeword_b200.detection import DetectorRecords, MultiModelDetector, StreamDetector
    a = StreamDetector(4096, BASE, WINDOW, COOLDOWN)
    a.set_cutoffs([3, 9], [0.6, 0.9])
    a.update(torch.from_numpy(_probs(4096, 40, 20)).cuda())
    rows = np.arange(0, 4096, 3)
    a.export_rows(rows).save(tmp_path / "plain.npz")
    b = StreamDetector(4096, BASE, WINDOW, COOLDOWN)
    b.import_rows(rows, DetectorRecords.load(tmp_path / "plain.npz", "cuda:0"))
    assert same_state(_rows(b.state_dict(), rows), _rows(a.state_dict(), rows))
    assert np.array_equal(b.cutoffs, np.where(np.isin(np.arange(4096), rows), a.cutoffs, BASE))
    S = 2048
    eng = _models_engine(S, [None, np.arange(0, S, 2, dtype=np.int32), None])
    m = MultiModelDetector(eng, **RULES)
    _feed(torch, m, [_probs(S, 20, 21), _probs(S, 20, 22), np.full((S, 20), 0.9, np.float32)], 0, 20)
    ids = np.arange(S)
    m.export_streams(ids).save(tmp_path / "multi.npz")
    n = MultiModelDetector(eng, **RULES)
    n.import_streams(ids, DetectorRecords.load(tmp_path / "multi.npz", "cuda:0"))
    for x, y in zip(n.state_dict()["models"], m.state_dict()["models"]):
        assert all(np.array_equal(x[f], y[f]) for f in x)


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200 import _lib
    from microwakeword_b200.detection import DetectorRecords, MultiModelDetector, StreamDetector
    a, b = StreamDetector(512, BASE, WINDOW, COOLDOWN), StreamDetector(512, BASE, WINDOW, COOLDOWN)
    for d, seed in ((a, 30), (b, 31)):
        d.set_cutoffs([1, 2], 0.6)
        d.update(torch.from_numpy(_probs(512, 20, seed)).cuda())
    snap = lambda: [(d.state_dict(), d.cutoffs) for d in (a, b)]
    before = snap()
    rec = a.export_rows([0, 1, 2, 3])
    L = _lib.lib()

    def refused(fn, *words):
        with pytest.raises(_lib.MwwError) as e:
            fn()
        assert e.value.code == -1 and all(w in str(e.value) for w in words), str(e.value)

    refused(lambda: a.export_rows([0, 512]), "out of range")
    refused(lambda: b.import_rows([0, -1, 2, 3], rec), "out of range")
    refused(lambda: b.import_rows([0, 1, 1, 3], rec), "listed twice")
    for det, field in ((StreamDetector(512, BASE, 4, COOLDOWN), "window"), (StreamDetector(512, BASE, WINDOW, 24), "cooldown_slices")):
        refused(lambda: det.import_rows([0, 1, 2, 3], rec), field)
    eng = _models_engine(512, None)
    m = MultiModelDetector(eng, **RULES)
    refused(lambda: m.import_streams([0, 1, 2, 3], rec), "multi")
    mrec = m.export_streams([0, 1])
    refused(lambda: b.import_rows([0, 1], mrec), "multi")
    bad = _lib.MwwDetectorLayout.from_buffer_copy(bytes(rec.layout))
    bad.record_bytes = 64
    refused(lambda: b.import_rows([0, 1, 2, 3], DetectorRecords(torch.zeros((4, 64), dtype=torch.uint8, device="cuda"), bad, rec.cutoffs)),
            "record_bytes")
    # the C calls' own checks: n < 0, misaligned or NULL records, a NULL layout
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ids = (ctypes.c_int32 * 2)(0, 1)
    buf = torch.zeros(4 * 48 + 16, dtype=torch.uint8, device="cuda")
    assert L.mww_export_detector_rows(a._d, ids, -1, buf.data_ptr(), None, st) == -1
    assert L.mww_export_detector_rows(a._d, ids, 2, buf.data_ptr() + 4, None, st) == -1 and b"aligned" in L.mww_last_error(None)
    assert L.mww_import_detector_rows(b._d, ids, 2, None, ctypes.byref(rec.layout), st) == -1
    assert L.mww_import_detector_rows(b._d, ids, 2, buf.data_ptr(), None, st) == -1 and b"layout" in L.mww_last_error(None)
    # n == 0: no device work, the layout still filled / checked
    lay = _lib.MwwDetectorLayout()
    assert L.mww_export_detector_rows(a._d, None, 0, None, ctypes.byref(lay), st) == 0 and lay.record_bytes == 48 and lay.role[0] == 1
    assert L.mww_import_detector_rows(b._d, None, 0, None, ctypes.byref(mrec.layout), st) == -1
    after = snap()
    for (s0, c0), (s1, c1) in zip(before, after):
        assert same_state(s0, s1) and np.array_equal(c0, c1)


# ---- launches and event buffers ---------------------------------------------------------------------------------------------------
def _kernels(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                  and "memset" not in e.name.lower())


def test_launch_count_does_not_depend_on_n(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import MultiModelDetector, StreamDetector
    src, dst = StreamDetector(R_SRC, BASE), StreamDetector(R_SRC, BASE)
    eng = _models_engine(R_SRC, [None, np.arange(0, R_SRC, 2, dtype=np.int32), None])
    m, m2 = MultiModelDetector(eng, **RULES), MultiModelDetector(eng, **RULES)
    for s, d, exp, imp in ((src, dst, "export_rows", "import_rows"), (m, m2, "export_streams", "import_streams")):
        seen = []
        for n in (1, R_SRC):
            ids = np.random.default_rng(n).permutation(R_SRC)[:n].astype(np.int32)
            rec = getattr(s, exp)(ids)
            e = _kernels(torch, lambda: getattr(s, exp)(ids))
            i = _kernels(torch, lambda: getattr(d, imp)(ids, rec))
            assert sum("pack_detector_rows_kernel" in k and "unpack" not in k for k in e) == 1, e
            assert sum("unpack_detector_rows_kernel" in k for k in i) == 1, i
            seen.append((len(e), len(i)))
        assert seen[0] == seen[1], seen


def test_export_and_import_leave_the_event_buffers_alone(torch_cuda):
    torch = torch_cuda
    from microwakeword_b200.detection import StreamDetector
    a, b = StreamDetector(1024, BASE, WINDOW, COOLDOWN), StreamDetector(1024, BASE, WINDOW, COOLDOWN)
    a.update(torch.from_numpy(_probs(1024, 40, 40)).cuda())
    b.update(torch.from_numpy(_probs(1024, 40, 41)).cuda())
    views = lambda: [(d.event_count.cpu().clone(), d.fired_ids.cpu().clone()) for d in (a, b)]
    v0 = views()
    assert int(v0[0][0]) > 0 and int(v0[1][0]) > 0
    b.import_rows(np.arange(0, 1024, 2), a.export_rows(np.arange(512)))
    torch.cuda.synchronize()
    v1 = views()
    assert all(torch.equal(x, y) for p, q in zip(v0, v1) for x, y in zip(p, q))
    ea, eb = _drain_all(a), _drain_all(b)
    assert ea.size == int(v0[0][0]) and eb.size == int(v0[1][0])
