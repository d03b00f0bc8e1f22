"""Second-stage verification on the GPU (run with -m gpu on an H100).

Every score and confirmed id is compared bit for bit with an independent path built from the existing public calls: the
source engine's audio_history of the ids, a newly created StreamEngine of the verifier's container, predict_clip,
detection.positive_scores and the cutoff, with NaN / -1 for ids that name no stream.  The live loop runs 4 099 streams of
the fp32 okay_nabu container on 480-sample step() calls with a 48 000-sample history, and a StreamDetector whose cutoff a
first pass sets so that some streams fire and most do not; it verifies at every drain with int8 okay_nabu, fp32 okay_nabu and
the `wide` run-time geometry of tests/generic_range.py, reusing each verifier.  For a few slots the CPU oracle
(oracle.run_pipeline, oracle/detection_ref.positive_score) scores the read-back audio: int8 bit for bit, fp32 within the
fp32 parity tolerance.  Also: a MultiModelDetector's per-model slots, a plain detector past its capacity, an 8 kHz mu-law
source against a 16 kHz one given the same history audio, that nothing of the source or the detector moves, launch counts
that do not depend on the number of events, a verify on a non-default CUDA stream, and the refusals.  Not exercised here:
the refusal of a source on another GPU (one GPU) and of a poisoned source (poisoning needs a failed staged call)."""

import ctypes
import os

import numpy as np
import pytest
import torch

import oracle
from bench import synth_audio_device
from conftest import GOLDEN
from generic_range import GEOMETRIES
from microwakeword_b200 import _lib
from microwakeword_b200 import model_file as MF
from microwakeword_b200.detection import MODEL_EVENT_DTYPE, MultiModelDetector, StreamDetector, positive_scores
from microwakeword_b200.engine import MultiModelEngine, StreamEngine
from microwakeword_b200.verify import Verifier
from oracle import detection_ref
from oracle import mixednet_ref as R

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5                      # tests/test_gpu_parity.py: fp32 probabilities against the oracle
S = 4099
HIST = 48000
N = 32000                           # 2 s: 198 frames, 66 okay_nabu steps
CUT = 0.5


def _blob(path):
    with open(path, "rb") as f:
        return f.read()


F32 = _blob(os.path.join(GOLDEN, "okay_nabu_synth_f32.mww"))
I8 = _blob(os.path.join(GOLDEN, "okay_nabu_synth_int8.mww"))


def wide_blob():
    spec = GEOMETRIES["wide"]
    return MF.write_container(R.fold_bn(spec, R.init_synthetic(spec, 0)))


def audio(n_streams, n_samples, seed):
    return synth_audio_device(torch, n_streams, n_samples, seed, torch.device("cuda", 0))


def reference(eng, ids, blob, n_samples=N, cutoff=CUT, window=5, ignore=25):
    """(scores, confirmed, audio) of the ids by the independent path"""
    ids_d = ids if isinstance(ids, torch.Tensor) else torch.tensor(np.asarray(ids, np.int32), device="cuda")
    a = eng.audio_history(ids_d, n_samples)
    h = ids_d.cpu().numpy()
    scores = np.full(h.size, np.nan, np.float32)
    confirmed = np.full(h.size, -1, np.int32)
    listed = np.nonzero((h >= 0) & (h < eng.n_streams))[0]
    if listed.size:
        fresh = StreamEngine(blob, n_streams=listed.size)
        probs = fresh.predict_clip(a[torch.from_numpy(listed).cuda()].contiguous())
        fresh.close()
        s = positive_scores(list(probs), window, ignore)
        scores[listed] = s
        confirmed[listed] = np.where(s.astype(np.float64) > cutoff, h[listed], -1)
    return scores, confirmed, a.cpu().numpy()


def same(got, want):
    """bit-identical float32 scores (NaN where NaN) and int32 ids"""
    gs, gc = (t.cpu().numpy() for t in got)
    ws, wc = want[:2]
    assert gs.shape == ws.shape and np.array_equal(np.isnan(gs), np.isnan(ws))
    ok = ~np.isnan(ws)
    assert np.array_equal(gs.view(np.uint32)[ok], ws.view(np.uint32)[ok])
    assert np.array_equal(gc, wc)


def live_cutoff(eng, chunks, quantile):
    """a detector cutoff from a first pass: the given quantile of each stream's largest 5-step average"""
    probs = torch.cat([eng.step(c) for c in chunks], 1)
    avg = probs.unfold(1, 5, 1).mean(2).amax(1).cpu().numpy()
    eng.reset()
    return float(np.quantile(avg, quantile))


def test_live_loop_against_the_independent_path_and_the_oracle():
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(HIST)
    calls, D = 160, 40
    x = audio(S, 480 * calls, 101)
    chunks = [x[:, 480 * i:480 * (i + 1)].contiguous() for i in range(calls)]
    cutoff = live_cutoff(eng, chunks[:80], 0.97)
    det = StreamDetector(S, cutoff, capacity=256)
    blobs = {"int8": I8, "f32": F32, "wide": wide_blob()}
    vers = {k: Verifier(b, slots=256, n_samples=N, cutoff=CUT) for k, b in blobs.items()}
    assert vers["f32"].steps == 66 and vers["int8"].steps == 66
    fired_total, drains_with_events, oracle_done = 0, 0, set()
    for i, c in enumerate(chunks):
        det.update(eng.step(c))
        if (i + 1) % D:
            continue
        n = int(det.event_count.item())
        fired_total += n
        drains_with_events += n > 0
        for k, ver in vers.items():
            want = reference(eng, det.fired_ids, blobs[k])
            same(ver.verify(eng, det.fired_ids), want)           # mww_verify_streams on the detector's d_fired
            same(ver.verify(eng, det), want)                     # mww_verify_detections: the same slots
            listed = np.nonzero(det.fired_ids.cpu().numpy() >= 0)[0][:4]
            if listed.size and k in ("int8", "f32") and k not in oracle_done:
                oracle_done.add(k)
                got = ver.verify(eng, det)[0].cpu().numpy()[listed]
                a = want[2][listed]
                _, p = oracle.run_pipeline(blobs[k], a, want_features=False)
                ref = np.asarray([detection_ref.positive_score(p[j, :66]) for j in range(listed.size)], np.float32)
                if k == "int8":
                    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
                else:
                    assert np.abs(got - ref).max() <= F32_TOL
        eng.reset(det.fired_ids)                                 # after verifying: a reset zeroes the history
        det.reset(det.fired_ids)
        det.drain()
    assert oracle_done == {"int8", "f32"}
    assert drains_with_events >= 2 and 0 < fired_total < S // 4
    for ver in vers.values():
        ver.close()


def test_multi_model_detector_slots_and_drain():
    Sm = 1024
    eng = MultiModelEngine([F32, I8, F32], n_streams=Sm)
    eng.set_audio_history(N)
    calls = 100
    x = audio(Sm, 480 * calls, 202)
    chunks = [x[:, 480 * i:480 * (i + 1)].contiguous() for i in range(calls)]
    first = [torch.cat(p, 1) for p in zip(*[eng.step(c) for c in chunks[:70]])]
    cut = [float(np.quantile(p.unfold(1, 5, 1).mean(2).amax(1).cpu().numpy(), 0.97)) for p in first]
    vad_cut = float(np.quantile(first[2].unfold(1, 5, 1).mean(2).cpu().numpy(), 0.05))
    eng.reset()
    det = MultiModelDetector(eng, cutoffs=[cut[0], cut[1], vad_cut], vad=2, capacity=512)
    for c in chunks:
        det.update(eng.step(c))
    ver = {k: Verifier(b, slots=512, n_samples=N, cutoff=CUT) for k, b in ((0, F32), (1, I8))}
    got = {k: ver[k].verify(eng, det, model=k) for k in ver}
    every = ver[0].verify(eng, det)                              # model None: every used slot
    n = int(det.event_count.item())
    ev, fired = det._drain_slots(MODEL_EVENT_DTYPE)
    assert fired == n and 0 < n <= 512 and set(ev["model"]) == {0, 1}
    for k in ver:
        ids = np.full(512, -1, np.int32)
        mine = np.nonzero(ev["model"] == k)[0]
        ids[mine] = ev["stream"][mine]
        same(got[k], reference(eng, ids, F32 if k == 0 else I8))
        assert np.isnan(got[k][0].cpu().numpy()[:n][ev["model"] != k]).all() and (got[k][1].cpu().numpy()[n:] == -1).all()
    ids = np.full(512, -1, np.int32)
    ids[:n] = ev["stream"]
    same(every, reference(eng, ids, F32))
    # Verifier.drain: the last verify's score of each event of its model, paired by slot; NaN for the other model's
    for c in chunks[:30]:
        det.update(eng.step(c))
    s0, _ = ver[0].verify(eng, det, model=0)
    slot_scores = s0.cpu().numpy()
    det.update(eng.step(chunks[30]))                             # may fire after the verify: those events have no score
    drained, dropped = ver[0].drain(det)
    assert dropped == 0 and drained.dtype.names[-1] == "verifier_score"
    assert np.array_equal(drained[["model", "step", "stream"]], np.sort(drained[["model", "step", "stream"]]))
    assert all(e["model"] == 0 for e in drained if not np.isnan(e["verifier_score"]))
    assert np.array_equal(np.sort(drained["verifier_score"][~np.isnan(drained["verifier_score"])]),
                          np.sort(slot_scores[~np.isnan(slot_scores)]))
    again, _ = ver[0].drain(det)                                 # nothing verified since: no scores
    assert again.size == 0 or np.isnan(again["verifier_score"]).all()
    for v in ver.values():
        v.close()


def test_plain_detector_past_its_capacity_verifies_the_first_slots():
    Sp = 512
    eng = StreamEngine(F32, n_streams=Sp)
    eng.set_audio_history(N)
    x = audio(Sp, 480 * 80, 303)
    det = StreamDetector(Sp, cutoff=-1.0, cooldown_slices=0, capacity=16)      # every row fires on every step
    for i in range(80):
        det.update(eng.step(x[:, 480 * i:480 * (i + 1)].contiguous()))
    assert int(det.event_count.item()) > 16
    ver = Verifier(F32, slots=16, n_samples=N, cutoff=CUT)
    same(ver.verify(eng, det), reference(eng, det.fired_ids, F32))
    assert (det.fired_ids.cpu().numpy() >= 0).all()
    ver.close()


def test_an_8khz_ulaw_source_scores_as_a_16khz_one_given_the_same_history():
    Ss = 256
    src = StreamEngine(F32, n_streams=Ss, stream_rates=[8000] * Ss)
    src.set_audio_history(N)
    g = torch.Generator(device="cuda").manual_seed(7)
    codes = torch.randint(0, 256, (Ss, 240 * 80), dtype=torch.uint8, device="cuda", generator=g)
    for i in range(80):
        src.step(codes[:, 240 * i:240 * (i + 1)].contiguous(), law="ulaw")
    ids = torch.randperm(Ss, device="cuda", generator=g)[:64].to(torch.int32)
    ids[::9] = -1
    heard = src.audio_history(torch.arange(Ss, dtype=torch.int32, device="cuda"), N)
    plain = StreamEngine(F32, n_streams=Ss)
    plain.set_audio_history(N)
    plain.predict_clip(heard.contiguous())
    assert torch.equal(plain.audio_history(ids, N), src.audio_history(ids, N))
    ver = Verifier(I8, slots=64, n_samples=N, cutoff=CUT)
    a, b = ver.verify(src, ids), ver.verify(plain, ids)
    same(a, (b[0].cpu().numpy(), b[1].cpu().numpy()))
    same(a, reference(src, ids, I8))
    ver.close()


def _snapshot(eng, det):
    torch.cuda.synchronize()
    all_ids = torch.arange(eng.n_streams, dtype=torch.int32, device="cuda")
    hist = eng.audio_history(all_ids, eng.audio_history_capacity).cpu().numpy()
    return dict(state=eng.state_dict(), hist=hist, seen=eng.audio_samples_seen, det=det.state_dict(),
                count=int(det.event_count.item()), fired=det.fired_ids.cpu().numpy().copy())


def _same_snapshot(a, b):
    for k in ("hist", "fired"):
        assert np.array_equal(a[k], b[k]), k
    assert a["seen"] == b["seen"] and a["count"] == b["count"]
    for part in ("state", "det"):
        assert a[part].keys() == b[part].keys()
        for k in a[part]:
            assert np.array_equal(np.asarray(a[part][k]), np.asarray(b[part][k])), (part, k)


def test_nothing_else_moves_and_launches_do_not_depend_on_events():
    Sn = 300
    eng = StreamEngine(F32, n_streams=Sn)
    eng.set_audio_history(N)
    x = audio(Sn, 480 * 70, 404)
    probs = [eng.step(x[:, 480 * i:480 * (i + 1)].contiguous()) for i in range(70)]
    dets = {"none": StreamDetector(Sn, cutoff=2.0, capacity=32), "one": StreamDetector(Sn, cutoff=2.0, cooldown_slices=40, capacity=32),
            "full": StreamDetector(Sn, cutoff=-1.0, capacity=32)}
    dets["one"].set_cutoffs([5], [-1.0])
    for d in dets.values():
        for p in probs:
            d.update(p)
    counts = {k: int(d.event_count.item()) for k, d in dets.items()}
    assert counts["none"] == 0 and counts["one"] == 1 and dets["one"].fired_ids.cpu().numpy()[0] == 5
    assert counts["full"] > 32
    ver = Verifier(I8, slots=32, n_samples=N, cutoff=CUT)
    ver_launches, src_launches = {}, {}
    for k, d in dets.items():
        before = _snapshot(eng, d)
        v0, s0 = ver.launch_count, eng.launch_count
        got = ver.verify(eng, d)
        torch.cuda.synchronize()
        ver_launches[k], src_launches[k] = ver.launch_count - v0, eng.launch_count - s0
        _same_snapshot(before, _snapshot(eng, d))
        same(got, reference(eng, d.fired_ids, I8))
    assert len(set(ver_launches.values())) == 1 and ver_launches["none"] > 0
    assert set(src_launches.values()) == {1}                    # the history read, src's own kernel
    # a verify on another CUDA stream right after a step on it, without a host synchronisation
    side = torch.cuda.Stream()
    ids = torch.arange(0, Sn, 10, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(side):
        eng.step(x[:, :480].contiguous())
        got = ver.verify(eng, ids)
    side.synchronize()
    same(got, reference(eng, ids, I8))


def test_refusals_leave_everything_unchanged():
    L = _lib.lib()
    Sr = 64
    eng = StreamEngine(F32, n_streams=Sr)
    eng.set_audio_history(N)
    x = audio(Sr, 480 * 70, 505)
    det = StreamDetector(Sr, cutoff=-1.0, capacity=8)
    for i in range(70):
        det.update(eng.step(x[:, 480 * i:480 * (i + 1)].contiguous()))
    ver = Verifier(F32, slots=8, n_samples=N, cutoff=CUT)
    before, launches = _snapshot(eng, det), ver.launch_count
    ids = torch.arange(8, dtype=torch.int32, device="cuda")
    out_s = torch.empty(16, dtype=torch.float32, device="cuda")
    out_c = torch.empty(16, dtype=torch.int32, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    no_hist = StreamEngine(F32, n_streams=Sr)
    short = StreamEngine(F32, n_streams=Sr)
    short.set_audio_history(N - 8)
    big = StreamDetector(Sr, cutoff=0.5, capacity=9)
    v, h = ver._v, eng._h
    for rc in (L.mww_verify_streams(v, no_hist._h, ids.data_ptr(), 8, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_streams(v, short._h, ids.data_ptr(), 8, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_streams(v, h, ids.data_ptr(), -1, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_streams(v, h, ids.data_ptr(), 9, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_streams(v, h, None, 8, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_streams(None, h, ids.data_ptr(), 8, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_detections(v, h, big._d, -1, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_detections(v, h, det._d, 1, out_s.data_ptr(), out_c.data_ptr(), st),
               L.mww_verify_detections(v, no_hist._h, det._d, -1, out_s.data_ptr(), out_c.data_ptr(), st)):
        assert rc == -1 and L.mww_last_error(None)
    assert ver.launch_count == launches                         # no refusal launched anything on the verifier
    # either output may be NULL
    assert L.mww_verify_streams(v, h, ids.data_ptr(), 8, None, out_c.data_ptr(), st) == 0
    assert L.mww_verify_detections(v, h, det._d, 0, out_s.data_ptr(), None, st) == 0
    torch.cuda.synchronize()
    _same_snapshot(before, _snapshot(eng, det))
    # create: a rule that leaves every score NaN, a frontend-only blob, a container that does not load
    rule = lambda n, w=5, ig=25: _lib.MwwVerifyRule(n, w, ig, 0, 0.5)   # noqa: E731
    out = ctypes.c_void_p()
    assert L.mww_verifier_create(F32, len(F32), 0, 4, ctypes.byref(rule(480 + 160 * 86)), ctypes.byref(out)) == -1   # 29 steps < 25 + 5
    assert b"NaN" in L.mww_last_error(None) and out.value is None
    assert L.mww_verifier_create(F32, len(F32), 0, 4, ctypes.byref(rule(480 + 160 * 89)), ctypes.byref(out)) == 0      # 30: one score
    assert L.mww_verifier_destroy(out) == 0
    assert L.mww_verifier_create(None, 0, 0, 4, ctypes.byref(rule(N)), ctypes.byref(out)) == -1 and b"frontend-only" in L.mww_last_error(None)
    junk = b"\0" * 64
    rc = L.mww_verifier_create(junk, len(junk), 0, 4, ctypes.byref(rule(N)), ctypes.byref(out))
    assert rc not in (0, -1) and out.value is None
    with pytest.raises(_lib.MwwError):
        Verifier(F32, slots=4, n_samples=480, cutoff=0.5)
    ver.close()
