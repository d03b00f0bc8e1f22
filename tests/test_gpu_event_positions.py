"""Event positions on the GPU (run with -m gpu on an H100): timed detectors, history reads that end at given positions, and
verification anchored at the event (include/mww.h, "event positions").

- A timed and an untimed twin of each detector kind, fed the same probabilities, give the same events and state bit for bit:
  live calls (1 step, the thread form) and clip calls (66 steps, the warp form), uniform and per-row cutoffs, and a models
  detector with a VAD and stream sets.  A timed update is one kernel launch, as an untimed one: the update is captured into a
  CUDA graph and the graph's kernel nodes are counted, which does not depend on a profiler session.
- Every event of a 4 099-stream live loop sits where the formula puts it with the engine's counters of the call it fired in,
  and the history read that ends there equals the audio the test fed, kept on the host on the 16 kHz axis.  A per-stream-rate
  engine (8 kHz beside 48 kHz, mu-law) gives the events, positions and reads of a 16 kHz twin fed its history.
- verify(..., at_event=True, post=p) equals an independent path: the fed audio's slice [e - n_samples, e), a new StreamEngine's
  predict_clip, detection.positive_scores and the cutoff, bit for bit, for an int8 and an fp32 verifier.
- The same audio verified at drains every D = 1, 7 and 33 calls gives each event the same score (post = 0, and post > 0 for
  events at least post old; younger ones match the clamped reference).
- Expired events give NaN / -1; the handles' launch counts equal those of the "now" verify at 0, 1 and capacity events; nothing of the source
  or the detector moves; a verify on a non-default CUDA stream."""

import ctypes
import os

import numpy as np
import pytest
import torch

from bench import synth_audio_device
from conftest import GOLDEN
from microwakeword_b200.detection import MultiModelDetector, StreamDetector, positive_scores
from microwakeword_b200.engine import MultiModelEngine, StreamEngine
from microwakeword_b200.verify import Verifier

pytestmark = pytest.mark.gpu

HOP, WIN = 160, 480
N = 32000
CUT = 0.5


def _blob(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


F32 = _blob("okay_nabu_synth_f32.mww")
I8 = _blob("okay_nabu_synth_int8.mww")


def audio(n_streams, n_samples, seed):
    return synth_audio_device(torch, n_streams, n_samples, seed, torch.device("cuda", 0))


def split(x, sizes):
    out, t = [], 0
    for n in sizes:
        out.append(x[:, t:t + n].contiguous())
        t += n
    return out


def quantile_cutoff(probs, q):
    p = torch.cat(probs, 1)
    return float(np.quantile(p.unfold(1, 5, 1).mean(2).amax(1).cpu().numpy(), q))


def captured_kernels(fn):
    """the kernel launches fn() enqueues, counted as the kernel nodes of a CUDA graph captured from it; the captured work then
    runs once, so fn() has its effect"""
    g = torch.cuda.CUDAGraph(keep_graph=True)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        fn()
    cu = ctypes.CDLL("libcuda.so.1")
    h, n = ctypes.c_void_p(int(g.raw_cuda_graph())), ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(h, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * max(n.value, 1))()
    assert cu.cuGraphGetNodes(h, nodes, ctypes.byref(n)) == 0
    kinds = []
    for i in range(n.value):
        t = ctypes.c_int(-1)
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(nodes[i]), ctypes.byref(t)) == 0
        kinds.append(t.value)
    g.replay()
    torch.cuda.synchronize()
    return sum(k == 0 for k in kinds)                           # CU_GRAPH_NODE_TYPE_KERNEL


def untimed_view(ev):
    """the events without their positions, as a sorted list (events of one call are in no particular slot order)"""
    names = [n for n in ev.dtype.names if n != "sample"]
    return sorted(tuple(e) for e in ev[names].tolist())


def same_state(a, b):
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            same_state(a[k], b[k])
    elif isinstance(a, list):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            same_state(x, y)
    elif a is None:
        assert b is None
    else:
        a, b = np.ascontiguousarray(np.atleast_1d(a)), np.ascontiguousarray(np.atleast_1d(b))
        assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def clock(eng, k=None):
    """the last_end of the call just made on the engine's counters, and step_samples"""
    S = eng.audio_samples_seen
    b = eng.frontend_buffered - (WIN - eng.hop)
    g = eng.pending_rows if k is None else eng.pending_rows[k]
    s = eng.stride if k is None else eng.stride[k]
    return S - b - eng.hop * g, eng.hop * s


@pytest.mark.parametrize("per_row", [False, True])
def test_plain_twins_are_bit_identical_in_both_forms(per_row):
    Sn = 1000
    sizes = [480] * 30 + [N] * 3 + [480] * 30
    x = audio(Sn, sum(sizes), 11)
    eng = StreamEngine(F32, n_streams=Sn)
    eng.set_audio_history(48000)
    cut = quantile_cutoff([eng.predict_clip(c) for c in split(x, sizes)], 0.7)
    eng.reset()
    plain, timed = StreamDetector(Sn, cut, capacity=8192), StreamDetector(Sn, cut, capacity=8192, timed=True)
    if per_row:
        rows = np.arange(0, Sn, 7)
        for d in (plain, timed):
            d.set_cutoffs(rows, cut - 0.05)
    fired = 0
    for i, c in enumerate(split(x, sizes)):
        p = eng.predict_clip(c)
        if i in (1, 30):                                       # a live call and a clip call: one launch each
            assert captured_kernels(lambda: plain.update(p)) == 1
            assert captured_kernels(lambda: timed.update(p, eng)) == 1
        else:
            plain.update(p)
            timed.update(p, eng)
        if i % 9 == 8:
            rows = plain.fired_ids[plain.fired_ids >= 0][:5].cpu().numpy()
            plain.reset(rows)
            timed.reset(rows)
        if i % 10 == 9 or i == len(sizes) - 1:
            a, na = plain.drain()
            b, nb = timed.drain()
            assert na == nb and a.dtype.names + ("sample",) == b.dtype.names
            assert untimed_view(a) == untimed_view(b)
            fired += a.size
            same_state(plain.state_dict(), timed.state_dict())
    assert fired > 50


def test_models_twins_are_bit_identical():
    Sm = 800
    sets = [np.arange(Sm), np.arange(0, Sm, 2), np.arange(Sm // 3, Sm)]
    eng = MultiModelEngine([F32, I8, F32], n_streams=Sm, streams=sets)
    eng.set_audio_history(48000)
    sizes = [480] * 25 + [N, 7520, N] + [480] * 25
    x = audio(Sm, sum(sizes), 12)
    first = [torch.cat(p, 1) for p in zip(*[eng.predict_clip(c) for c in split(x, sizes)])]
    cut = [float(np.quantile(p.unfold(1, 5, 1).mean(2).amax(1).cpu().numpy(), 0.6)) for p in first]
    vad_cut = float(np.quantile(first[2].unfold(1, 5, 1).mean(2).cpu().numpy(), 0.1))
    eng.reset()
    kw = dict(cutoffs=[cut[0], cut[1], vad_cut], vad=2, capacity=8192)
    plain, timed = MultiModelDetector(eng, **kw), MultiModelDetector(eng, timed=True, **kw)
    for d in (plain, timed):
        d.set_cutoffs(1, sets[1][::5], cut[1] - 0.05)
    fired = 0
    for i, c in enumerate(split(x, sizes)):
        p = eng.predict_clip(c)
        if i in (1, 25):
            assert captured_kernels(lambda: plain.update(p)) == 1
            assert captured_kernels(lambda: timed.update(p)) == 1
        else:
            plain.update(p)
            timed.update(p)
        if i % 10 == 9 or i == len(sizes) - 1:
            a, _ = plain.drain()
            b, _ = timed.drain()
            assert untimed_view(a) == untimed_view(b)
            fired += a.size
            same_state(plain.state_dict(), timed.state_dict())
    assert fired > 20


def host_slice(xh, ids, ends, n):
    """rows [e - n, e) of the host audio on the 16 kHz axis, zeros outside [max(0, S - C), S)"""
    ids, ends = np.asarray(ids, np.int64), np.asarray(ends, np.int64)
    t = ends[:, None] - n + np.arange(n)[None, :]
    ok = (t >= 0) & (t < xh.shape[1])
    out = np.zeros((ids.size, n), np.int16)
    out[ok] = xh[np.broadcast_to(ids[:, None], t.shape)[ok], t[ok]]
    return out


def test_positions_are_the_formula_and_reads_end_there():
    S, calls, C = 4099, 90, 48000
    x = audio(S, 480 * calls, 21)
    xh = x.cpu().numpy()
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(C)
    chunks = split(x, [480] * calls)
    cut = quantile_cutoff([eng.step(c) for c in chunks[:40]], 0.9)
    eng.reset()
    eng.set_audio_history(C)                                    # a new axis: sample t is sample t of x
    det = StreamDetector(S, cut, capacity=4096, timed=True)
    n_ev, checked = 0, 0
    for i, c in enumerate(chunks):
        det.update(eng.step(c), eng)
        want, _ = clock(eng)
        if i % 11 == 5:
            got = eng.audio_history(det.fired_ids, 4000, end=det.event_samples).cpu().numpy()
            ids, ends = det.fired_ids.cpu().numpy(), det.event_samples.cpu().numpy()
            used = ids >= 0
            assert np.array_equal(got[~used], np.zeros_like(got[~used]))
            assert np.array_equal(got[used], host_slice(xh, ids[used], ends[used], 4000))
            checked += used.sum()
        ev, _ = det.drain()
        assert (ev["sample"] == want).all()                     # a live call has one step: every event sits at last_end
        n_ev += ev.size
    assert n_ev > 20 and checked > 0
    # host ends, and ends outside the ring
    Sseen = eng.audio_samples_seen
    ends = [Sseen - 100, Sseen + 50, -1, Sseen - C + 3, 480 * 10]
    got = eng.audio_history([1, 2, 3, 4, 5], 800, end=ends).cpu().numpy()
    want = host_slice(xh, [1, 2, 3, 4, 5], ends, 800)
    want[:, :][np.arange(800)[None, :] + np.asarray(ends)[:, None] - 800 < Sseen - C] = 0
    assert np.array_equal(got, want)


def test_per_stream_rates_match_a_16khz_twin():
    Sr, calls = 512, 60
    rates = np.where(np.arange(Sr) % 2 == 0, 8000, 48000)
    src = StreamEngine(F32, n_streams=Sr, stream_rates=rates)
    twin = StreamEngine(F32, n_streams=Sr)
    for e in (src, twin):
        e.set_audio_history(16000)
    g = torch.Generator(device="cuda").manual_seed(5)
    width = 1440
    codes = torch.randint(0, 256, (Sr, width * calls), dtype=torch.uint8, device="cuda", generator=g)
    first = []
    probe = StreamEngine(F32, n_streams=Sr, stream_rates=rates)
    for i in range(calls):
        first.append(probe.predict_clip(codes[:, width * i:width * (i + 1)].contiguous(), samples16=480, law="ulaw"))
    cut = quantile_cutoff(first, 0.8)
    d_src, d_twin = (StreamDetector(Sr, cut, capacity=2048, timed=True) for _ in range(2))
    all_ids = torch.arange(Sr, dtype=torch.int32, device="cuda")
    n_ev = 0
    for i in range(calls):
        p = src.predict_clip(codes[:, width * i:width * (i + 1)].contiguous(), samples16=480, law="ulaw")
        heard = src.audio_history(all_ids, 480).contiguous()
        q = twin.predict_clip(heard)
        assert torch.equal(p, q)
        d_src.update(p, src)
        d_twin.update(q, twin)
        if i % 10 == 9:
            ea, _ = d_src.drain()
            eb, _ = d_twin.drain()
            assert np.array_equal(ea, eb)
            if ea.size:
                a = src.audio_history(ea["stream"], 2400, end=ea["sample"])
                assert torch.equal(a, twin.audio_history(eb["stream"], 2400, end=eb["sample"]))
                assert a.abs().sum() > 0
            n_ev += ea.size
    assert n_ev > 0


def reference_at(xh, ids, ends, blob, n=N, cutoff=CUT):
    """(scores, confirmed) of slots (id, end) by the independent path on the host audio; id -1: NaN / -1"""
    ids, ends = np.asarray(ids), np.asarray(ends)
    scores = np.full(ids.size, np.nan, np.float32)
    confirmed = np.full(ids.size, -1, np.int32)
    listed = np.nonzero(ids >= 0)[0]
    if listed.size:
        a = torch.from_numpy(host_slice(xh, ids[listed], ends[listed], n)).cuda()
        fresh = StreamEngine(blob, n_streams=listed.size)
        probs = fresh.predict_clip(a)
        fresh.close()
        s = positive_scores(list(probs), 5, 25)
        scores[listed] = s
        confirmed[listed] = np.where(s.astype(np.float64) > cutoff, ids[listed], -1)
    return scores, confirmed


def same(got, want):
    gs, gc = (t.cpu().numpy() for t in got)
    ws, wc = want
    assert np.array_equal(np.isnan(gs), np.isnan(ws))
    ok = ~np.isnan(ws)
    assert np.array_equal(gs.view(np.uint32)[ok], ws.view(np.uint32)[ok])
    assert np.array_equal(gc, wc)


def slots(det, post, S, C, n=N):
    """the (id, end) of each slot the rule gives, from the detector's device views"""
    ids, pos = det.fired_ids.cpu().numpy().copy(), det.event_samples.cpu().numpy()
    e = np.minimum(pos + post, S)
    ids[(ids >= 0) & (e - n < S - C)] = -1
    return ids, np.where(ids >= 0, e, -1)


def run_polled(x, xh, D, cut, blobs, post, C=48000, Sn=512):
    eng = StreamEngine(F32, n_streams=Sn)
    eng.set_audio_history(C)
    det = StreamDetector(Sn, cut, capacity=1024, timed=True)
    vers = {k: Verifier(b, slots=1024, n_samples=N, cutoff=CUT) for k, b in blobs.items()}
    out = {}
    calls = x.shape[1] // 480
    for i in range(calls):
        det.update(eng.step(x[:, 480 * i:480 * (i + 1)].contiguous()), eng)
        if (i + 1) % D and i != calls - 1:
            continue
        S = eng.audio_samples_seen
        ids, ends = slots(det, post, S, C)
        pos, fired = det.event_samples.cpu().numpy(), det.fired_ids.cpu().numpy()
        for k, ver in vers.items():
            got = ver.verify(eng, det, at_event=True, post=post)
            same(got, reference_at(xh, ids, ends, blobs[k]))
            gs, gc = (t.cpu().numpy() for t in got)
            for j in np.nonzero(fired >= 0)[0]:
                out[(k, int(fired[j]), int(pos[j]))] = (gs[j], gc[j], S - pos[j])
        det.drain()
    for v in vers.values():
        v.close()
    return out


def test_anchored_verify_is_the_independent_path_and_does_not_depend_on_the_poll():
    Sn, calls = 512, 99
    x = audio(Sn, 480 * calls, 31)
    xh = x.cpu().numpy()
    probe = StreamEngine(F32, n_streams=Sn)
    cut = quantile_cutoff([probe.step(x[:, 480 * i:480 * (i + 1)].contiguous()) for i in range(calls)], 0.8)
    blobs = {"int8": I8, "f32": F32}
    for post in (0, 3200):
        runs = {D: run_polled(x, xh, D, cut, blobs, post) for D in (1, 7, 33)}
        keys = set(runs[1])
        assert len(keys) > 10 and all(set(r) == keys for r in runs.values())
        for key in keys:
            old = [r[key] for r in runs.values() if r[key][2] >= post]
            for a in old[1:]:                                  # every event at least post old: one score, whatever D
                assert np.array_equal(np.float32(a[0]).view(np.uint32), np.float32(old[0][0]).view(np.uint32)) or \
                    (np.isnan(a[0]) and np.isnan(old[0][0]))
                assert a[1] == old[0][1]
        if post == 0:
            assert all(r[key][2] >= 0 for r in runs.values() for key in keys)


def _snapshot(eng, det):
    torch.cuda.synchronize()
    all_ids = torch.arange(eng.n_streams, dtype=torch.int32, device="cuda")
    return dict(state=eng.state_dict(), hist=eng.audio_history(all_ids, eng.audio_history_capacity).cpu().numpy(),
                seen=eng.audio_samples_seen, det=det.state_dict(), count=int(det.event_count.item()),
                fired=det.fired_ids.cpu().numpy().copy(), pos=det.event_samples.cpu().numpy().copy())


def test_expiry_launches_side_effects_and_streams():
    Sn, C = 300, N + 8                                          # a ring just longer than the clip: events expire fast
    x = audio(Sn, 480 * 90, 41)
    xh = x.cpu().numpy()
    eng = StreamEngine(F32, n_streams=Sn)
    eng.set_audio_history(C)
    dets = {"none": StreamDetector(Sn, cutoff=2.0, capacity=32, timed=True),
            "one": StreamDetector(Sn, cutoff=2.0, cooldown_slices=40, capacity=32, timed=True),
            "full": StreamDetector(Sn, cutoff=-1.0, capacity=32, timed=True)}
    dets["one"].set_cutoffs([5], [-1.0])
    for i in range(70):
        p = eng.step(x[:, 480 * i:480 * (i + 1)].contiguous())
        for d in dets.values():
            d.update(p, eng)
    ver = Verifier(I8, slots=32, n_samples=N, cutoff=CUT)
    for k, d in dets.items():
        before = _snapshot(eng, d)
        # the verifier handle's launches and the source's (its history read) are counted by the handles; beside them both calls
        # run one slots kernel and one confirm kernel of the verifier's own
        v0, s0 = ver.launch_count, eng.launch_count
        ver.verify(eng, d)
        torch.cuda.synchronize()
        v1, s1 = ver.launch_count, eng.launch_count
        ver.verify(eng, d, at_event=True, post=480)
        torch.cuda.synchronize()
        assert v1 - v0 == ver.launch_count - v1 > 0 and s1 - s0 == eng.launch_count - s1 == 1, k
        got = ver.verify(eng, d, at_event=True, post=480)
        after = _snapshot(eng, d)
        for f in ("hist", "fired", "pos"):
            assert np.array_equal(before[f], after[f])
        assert before["seen"] == after["seen"] and before["count"] == after["count"]
        same_state(before["det"], after["det"])
        same_state(before["state"], after["state"])
        ids, ends = slots(d, 480, eng.audio_samples_seen, C)
        same(got, reference_at(xh, ids, ends, I8))
    # "full" fired on its first steps; 20 calls later their clips have left the ring
    d = dets["full"]
    for i in range(70, 90):
        eng.step(x[:, 480 * i:480 * (i + 1)].contiguous())
    s, c = ver.verify(eng, d, at_event=True, post=0)
    assert np.isnan(s.cpu().numpy()).all() and (c.cpu().numpy() == -1).all()
    # a verify on another CUDA stream right after a step on it, without a host synchronisation
    e2 = StreamEngine(F32, n_streams=Sn)
    e2.set_audio_history(48000)
    d2 = StreamDetector(Sn, cutoff=-1.0, capacity=32, timed=True)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for i in range(70):
            d2.update(e2.step(x[:, 480 * i:480 * (i + 1)].contiguous()), e2)
        got = ver.verify(e2, d2, at_event=True, post=960)
    side.synchronize()
    ids, ends = slots(d2, 960, e2.audio_samples_seen, 48000)
    same(got, reference_at(xh, ids, ends, I8))
    with pytest.raises(ValueError):
        ver.verify(eng, StreamDetector(Sn, cutoff=0.5), at_event=True)
    ver.close()


def test_refusals_leave_the_detector_unchanged():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    Sn = 64
    eng = StreamEngine(F32, n_streams=Sn)
    eng.set_audio_history(N)
    x = audio(Sn, 480 * 10, 51)
    probs = [eng.step(x[:, 480 * i:480 * (i + 1)].contiguous()) for i in range(10)]
    det = StreamDetector(Sn, cutoff=-1.0, capacity=64)
    det.update(probs[1])                                        # events buffered: timing is refused
    before = (det.state_dict(), int(det.event_count.item()), det.fired_ids.cpu().numpy().copy())
    assert L.mww_time_detector_events(det._d) == -1 and b"after create or a drain" in L.mww_last_error(None)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.mww_update_detector_at(det._d, probs[2].data_ptr(), 1, 1, 0, 160, st) == -1 and b"not timed" in L.mww_last_error(None)
    ver = Verifier(I8, slots=64, n_samples=N, cutoff=CUT)
    assert L.mww_verify_detections_at(ver._v, eng._h, det._d, -1, 0, None, None, st) == -1 and b"not timed" in L.mww_last_error(None)
    same_state(before[0], det.state_dict())
    assert before[1] == int(det.event_count.item()) and np.array_equal(before[2], det.fired_ids.cpu().numpy())
    det.drain()
    det._time()                                                 # after a drain: accepted
    before = (det.state_dict(), int(det.event_count.item()))
    assert L.mww_detector_update(det._d, probs[2].data_ptr(), 1, 1, st) == -1 and b"mww_update_detector_at" in L.mww_last_error(None)
    assert L.mww_update_detector_at(det._d, probs[2].data_ptr(), 1, 1, 0, 0, st) == -1 and b"step_samples" in L.mww_last_error(None)
    for post in (-1, 2 ** 22 + 1):
        assert L.mww_verify_detections_at(ver._v, eng._h, det._d, -1, post, None, None, st) == -1 and b"post" in L.mww_last_error(None)
    same_state(before[0], det.state_dict())
    assert before[1] == int(det.event_count.item()) == 0
    with pytest.raises(ValueError, match="audio history"):
        det.update(probs[3], StreamEngine(F32, n_streams=Sn))
    ver.close()
