"""Moving a stream's serving state between handles on the H100: the audio history write (mww_write_audio_history) against
the engine's own history reads, at 65 536 streams into handles of other sizes and capacities; the whole move a server makes
while commands are being spoken (stream records with history, detector rows and endpointer rows, in batches of ids) against
the source left in place as the stay-put reference, events and command clips bit for bit with positions shifted onto the
destination's axis; the truncated replay of a young destination endpointer against tests/endpoint_ref.py; a models engine
whose VAD model serves a subset of streams, into another stream set; one launch per call at n = 1 and n = 65 536; and every
refusal of the C-ABI, which leaves the state, the history and the launch counts unchanged.  The endpointers are fed
scripted speech probabilities (speech bursts and pauses) of the calls' real step counts, placed by the handles' real
counters; the audio is synth_audio's."""

import ctypes
import os

import numpy as np
import pytest

import endpoint_ref as R
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

F32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
RULE = dict(vad_window=5, vad_cutoff=0.5, speech_steps=3, silence_steps=8, timeout_steps=100, max_steps=120, lookback_steps=12)


def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _write(eng, ids, rows, n_samples=None, stride=None, ptr=None):
    """mww_write_audio_history on host ids -> return code"""
    ids = np.ascontiguousarray(ids, np.int32)
    n_samples = rows.shape[1] if n_samples is None else n_samples
    stride = (rows.stride(0) if rows.shape[0] > 1 else max(rows.shape[1], 1)) if stride is None else stride
    p = (rows.data_ptr() if rows.numel() else None) if ptr is None else ptr
    return eng._L.mww_write_audio_history(eng._h, ids.ctypes.data, ids.size, n_samples, p, stride, _stream())


def _audio_bank(P, n, seed):
    """P distinct synthetic streams of n samples on the GPU"""
    import torch
    from microwakeword_b200.synth_audio import synth_audio
    return torch.from_numpy(np.stack([synth_audio(n, seed + i) for i in range(P)])).cuda()


def _streams_audio(bank, S, call, salt=0):
    """[S, 480] of call `call`: stream s plays bank row (s * 7 + salt) % P, from an offset of its own"""
    import torch
    P, n = bank.shape
    s = torch.arange(S, device="cuda")
    row = (s * 7 + salt) % P
    off = (s * 131 + 480 * call) % (n - 480)
    idx = off[:, None] + torch.arange(480, device="cuda")[None, :]
    return bank[row[:, None], idx].contiguous()


# ---- the history write ------------------------------------------------------------------------------------------------------------
def test_history_round_trip_65536_streams_into_other_sizes_and_capacities():
    import torch
    from microwakeword_b200.engine import StreamEngine
    S, C = 65536, 32000
    src = StreamEngine(F32, n_streams=S)
    src.set_audio_history(C)
    bank = _audio_bank(61, 16000 * 8, 10)
    for c in range(80):                                             # 38 400 samples: the ring wrapped
        src.step(_streams_audio(bank, S, c))
    rng = np.random.default_rng(0)
    ids = np.concatenate([[0, S - 1], rng.choice(np.arange(1, S - 1), 1022, replace=False)]).astype(np.int32)
    for Cd, Sd in ((16000, 40960), (64000, 70000)):
        dst = StreamEngine(F32, n_streams=Sd)
        dst.set_audio_history(Cd)
        dst.predict_clip(_streams_audio(bank, Sd, 3, salt=5)[:, :477].contiguous())   # an odd axis: the scalar form
        for c in range(7):
            dst.step(_streams_audio(bank, Sd, c, salt=9))
        for n in (0, 8, 4801, C):
            to = rng.permutation(Sd)[:ids.size].astype(np.int32)
            rows = src.audio_history(ids, n)
            before = dst.audio_history(np.arange(Sd), Cd).clone()
            L0 = dst.launch_count
            assert _write(dst, to, rows) == 0
            assert dst.launch_count - L0 == 1                        # one launch whatever n is
            after = dst.audio_history(np.arange(Sd), Cd)
            m = min(n, Cd)
            want = torch.zeros((ids.size, Cd), dtype=torch.int16, device="cuda")
            if m:
                want[:, Cd - m:] = rows[:, n - m:]
            assert torch.equal(after[torch.from_numpy(to).long().cuda()], want), (Cd, n)
            keep = torch.ones(Sd, dtype=torch.bool, device="cuda")
            keep[torch.from_numpy(to).long().cuda()] = False
            assert torch.equal(after[keep], before[keep])           # every other row's bytes unchanged
            del before, after
            # 20 more identical calls on both handles: the histories still agree
            for c in range(20):
                a = _streams_audio(bank, S, 100 + c)
                b = _streams_audio(bank, Sd, 100 + c, salt=3)
                b[torch.from_numpy(to).long().cuda()] = a[torch.from_numpy(ids).long().cuda()]
                src.step(a)
                dst.step(b)
            k = min(n + 20 * 480, Cd, C)
            assert torch.equal(dst.audio_history(to, k), src.audio_history(ids, k)), (Cd, n)
        dst.close()


# ---- the headline: a move while commands are being spoken --------------------------------------------------------------------------
def _script(S, steps, rng):
    """speech probabilities [S, steps] by class of s % 4: bursts and pauses, constant speech (commands that run to
    max_steps), one burst just before the move, noise around the cutoff"""
    j = np.arange(steps)[None, :]
    period = rng.integers(3, 14, S)[:, None]
    phase = rng.integers(0, 40, S)[:, None]
    bursts = np.where(((j + phase) // period) % 2 == 0, 0.9, 0.05)
    one = np.where((j >= 185) & (j < 194), 0.95, 0.02) + 0 * phase
    noise = rng.uniform(0.3, 0.7, (S, steps))
    cls = (np.arange(S) % 4)[:, None]
    p = np.where(cls == 0, bursts, np.where(cls == 1, 0.9, np.where(cls == 2, one, noise)))
    return p.astype(np.float32)


def _sorted(ev):
    return ev[np.lexsort((ev["stream"], ev["end_sample"]))]


def test_move_while_commands_are_spoken_matches_the_stay_put_reference():
    import torch
    from microwakeword_b200.detection import StreamDetector
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S, Sd, C = 65536, 98304, 64000
    PRE, POST, MAX, CAP = 1600, 3200, 64000, 8192
    BEFORE, AFTER, DST_BEFORE = 200, 130, 70
    rng = np.random.default_rng(1)
    bank = _audio_bank(97, 16000 * 30, 100)
    P = _script(S, BEFORE + AFTER, rng)
    src = StreamEngine(F32, n_streams=S)
    src.set_audio_history(C)
    ep = Endpointer(src, capacity=CAP, **RULE)
    det = StreamDetector(S, cutoff=0.9)
    arms = {99: rng.choice(np.arange(1, S, 4), 1000, replace=False),        # constant speech: commands older than the destination
            149: rng.choice(S, 1000, replace=False), 184: rng.choice(S, 1000, replace=False), 194: rng.choice(S, 1000, replace=False),
            209: rng.choice(S, 1000, replace=False), 239: rng.choice(np.arange(2, S, 4), 1000, replace=False),
            269: rng.choice(S, 1000, replace=False)}
    ended_before_move = used = 0
    for c in range(BEFORE):
        pr = src.step(_streams_audio(bank, S, c))
        det.update(pr)
        n = pr.shape[1]                                              # the call's real step count (0 on the first call)
        ep.update(torch.from_numpy(P[:, used:used + n]).cuda())
        used += n
        if c % 5 == 4:
            ev, dropped = ep.drain()
            assert dropped == 0
            if c == BEFORE - 1:
                ended_before_move = ev.size                         # rows that ended just before the move
            det.drain()
        if c in arms:
            ep.arm(arms[c])
    st = ep.state_dict()
    armed = st["armed"] >= 0
    assert ended_before_move > 0
    assert (armed & (st["heard"] == 1) & (st["silence"] > 0)).sum() > 0      # armed mid-command, silence counting
    assert ((~armed) & ((st["flags"] & np.uint64(0xFFFF)) != 0)).sum() > 0   # unarmed with recent speech flags
    # the destination: a bigger handle whose endpointer has run >= 64 calls on its own streams
    dst = StreamEngine(F32, n_streams=Sd)
    dst.set_audio_history(C)
    dep = Endpointer(dst, capacity=CAP, **RULE)
    ddet = StreamDetector(Sd, cutoff=0.9)
    for c in range(DST_BEFORE):
        pr = dst.step(_streams_audio(bank, Sd, c, salt=11))
        ddet.update(pr)
        dep.update(torch.rand((Sd, pr.shape[1]), device="cuda"))
    dep.drain()
    ddet.drain()
    # the move: every stream, permuted ids, in batches of ids (the history buffer stays bounded)
    to = rng.permutation(Sd)[:S].astype(np.int32)
    shift = dst.audio_samples_seen - src.audio_samples_seen
    assert shift < 0
    ids = np.arange(S, dtype=np.int32)
    for b in range(0, S, 16384):
        recs = src.export_streams(ids[b:b + 16384], history=C)
        dst.import_streams(to[b:b + 16384], recs)
        del recs
    ddet.import_rows(to, det.export_rows(ids))
    L0 = dep.launch_count
    dep.import_streams(to, ep.export_streams(ids))
    assert dep.launch_count - L0 == 1
    to_t = torch.from_numpy(to).long().cuda()
    got_ev, want_ev = [], []
    negative = 0
    for c in range(BEFORE, BEFORE + AFTER):
        a = _streams_audio(bank, S, c)
        b = _streams_audio(bank, Sd, c, salt=13)
        b[to_t] = a
        pr, prd = src.step(a), dst.step(b)
        det.update(pr)
        ddet.update(prd)
        n = pr.shape[1]
        assert prd.shape[1] == n
        ps = torch.from_numpy(P[:, used:used + n]).cuda()
        used += n
        pd = torch.rand((Sd, n), device="cuda") * 0.4                 # the destination's own streams stay quiet
        pd[to_t] = ps
        ep.update(ps)
        dep.update(pd)
        if c % 5 == 4:
            clips, lens = ep.commands(PRE, POST, MAX)
            dclips, dlens = dep.commands(PRE, POST, MAX)
            torch.cuda.synchronize()
            ev, n = ep._drain_slots()
            dev_, dn = dep._drain_slots()
            assert n == dn and n <= CAP
            slot = {int(s): i for i, s in enumerate(dev_["stream"])}
            assert len(slot) == dn                                   # a stream ends at most once between arms
            j = torch.tensor([slot[int(to[s])] for s in ev["stream"]], dtype=torch.long, device="cuda")
            if ev.size:                                              # slot i of the source is slot j[i] of the destination
                assert torch.equal(lens[:ev.size], dlens[j]) and torch.equal(clips[:ev.size], dclips[j]), c
            m = ev.copy()
            m["stream"] = to[ev["stream"]]
            for k in ("start_sample", "end_sample", "speech_end_sample"):
                m[k] += shift
            want_ev.append(m)
            got_ev.append(dev_)
            negative += int((dev_["start_sample"] < 0).sum())
            del clips, dclips
        if c in arms:
            ep.arm(arms[c])
            dep.arm(to[arms[c]])
    want, got = _sorted(np.concatenate(want_ev)), _sorted(np.concatenate(got_ev))
    assert want.size > 1000 and np.array_equal(got, want)
    assert negative > 0                                              # positions before the destination's axis began


# ---- a young destination: the replay reaches back only as far as the rule says ---------------------------------------------------------
def _ref_of(ep, st, n_streams, members, rule):
    ref = R.EndpointRef(n_streams, members, ep.stride, ep.hop, capacity=ep.capacity, **rule)
    ref.hist = st["hist"].copy()
    for k in R.ROW_FIELDS:
        ref.rows[k] = st[k].astype(np.uint64 if k == "flags" else np.int64)
    ref.base = (st["samples_seen"], st["buffered"], st["pending"])
    ref.steps = st["steps"]
    ref.positions = [int(st["positions"][i]) for i in reversed(range(min(ref.steps, 64)))]
    ref.steps = len(ref.positions)
    return ref


def test_young_destination_replays_the_truncated_depth():
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S, Sd = 2048, 3000
    rule = dict(RULE, lookback_steps=40, timeout_steps=200, max_steps=300)
    rng = np.random.default_rng(2)
    P = _script(S, 80, rng)
    src, dst = StreamEngine(F32, n_streams=S), StreamEngine(F32, n_streams=Sd)
    src.set_audio_history(4800)
    dst.set_audio_history(4800)
    ep = Endpointer(src, capacity=S, **rule)
    dep = Endpointer(dst, capacity=S, **rule)
    bank = _audio_bank(13, 16000 * 4, 7)
    used = 0
    for c in range(60):
        n = src.step(_streams_audio(bank, S, c)).shape[1]
        ep.update(torch.from_numpy(P[:, used:used + n]).cuda())
        used += n
    for c in range(11):                                              # fewer steps than lookback_steps
        dep.update(torch.rand((Sd, dst.step(_streams_audio(bank, Sd, c)).shape[1]), device="cuda"))
    to = rng.permutation(Sd)[:S].astype(np.int32)
    dep.import_streams(to, ep.export_streams(np.arange(S)))
    torch.cuda.synchronize()
    ref = _ref_of(dep, dep.state_dict(), Sd, np.arange(Sd), rule)
    assert ref.steps == 10
    dep.arm(to)
    ref.arm(to)
    ep.arm(np.arange(S))
    got, want = dep.state_dict(), ref.state()
    for k in R.ROW_FIELDS:
        assert np.array_equal(got[k].astype(np.int64) if k != "flags" else got[k], want[k].astype(np.int64) if k != "flags" else want[k]), k
    assert np.array_equal(got["hist"].view(np.uint32), want["hist"].view(np.uint32))
    (ge, _), (re_, _) = dep.drain(), ref.drain()
    assert np.array_equal(_sorted(ge), _sorted(re_))
    # the source replayed 40 steps: the destination's elapsed is capped at its 10
    s_el = ep.state_dict()["elapsed"]
    assert got["elapsed"][to].max() <= 10 and s_el.max() > 10


# ---- a models engine: the VAD model on a subset, into another stream set -------------------------------------------------------------------
def test_models_engine_vad_subset_into_another_stream_set():
    import torch
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import MultiModelEngine
    S, Sd = 4096, 5000
    rng = np.random.default_rng(3)
    sub_s = np.flatnonzero(rng.random(S) < 0.5).astype(np.int32)
    sub_d = np.flatnonzero(rng.random(Sd) < 0.5).astype(np.int32)
    src = MultiModelEngine([F32, F32], n_streams=S, streams=[None, sub_s])
    dst = MultiModelEngine([F32, F32], n_streams=Sd, streams=[None, sub_d])
    for e in (src, dst):
        e.set_audio_history(4800)
    ep, dep = Endpointer(src, model=1, **RULE), Endpointer(dst, model=1, **RULE)
    P = _script(sub_s.size, 40, rng)
    bank = _audio_bank(13, 16000 * 2, 3)
    used = 0
    for c in range(40):
        n = src.predict_clip(_streams_audio(bank, S, c))[1].shape[1]
        ep.update(torch.from_numpy(P[:, used:used + n]).cuda())
        used += n
        if c == 25:
            ep.arm(sub_s[::3])
    for c in range(12):
        n = dst.predict_clip(_streams_audio(bank, Sd, c))[1].shape[1]
        dep.update(torch.rand((sub_d.size, n), device="cuda"))
    to = rng.permutation(Sd)[:S].astype(np.int32)
    s0, d0 = ep.state_dict(), dep.state_dict()
    shift = dst.audio_samples_seen - src.audio_samples_seen
    dep.import_streams(to, ep.export_streams(np.arange(S)))
    d1 = dep.state_dict()
    row_s = np.full(S, -1)
    row_s[sub_s] = np.arange(sub_s.size)
    row_d = np.full(Sd, -1)
    row_d[sub_d] = np.arange(sub_d.size)
    taken = fresh = 0
    touched = np.zeros(sub_d.size, bool)
    for s in range(S):
        r = row_d[to[s]]
        if r < 0:
            continue
        touched[r] = True
        q = row_s[s]
        if q < 0:
            fresh += 1
            assert d1["armed"][r] == -1 and d1["seen"][r] == 0 and d1["flags"][r] == 0 and not d1["hist"][r].any()
            continue
        taken += 1
        assert d1["seen"][r] == s0["seen"][q] and d1["flags"][r] == s0["flags"][q]
        assert np.array_equal(d1["hist"][r].view(np.uint32), s0["hist"][q].view(np.uint32))
        if s0["armed"][q] >= 0:
            assert d1["armed"][r] == to[s]
            for k in ("elapsed", "run", "silence", "heard"):
                assert d1[k][r] == s0[k][q], k
            for k in ("start_sample", "speech_end_sample"):
                assert d1[k][r] == s0[k][q] + shift, k
        else:
            assert d1["armed"][r] == -1 and d1["elapsed"][r] == 0 and d1["start_sample"][r] == 0
    assert taken > 0 and fresh > 0
    for k in ("seen", "flags", "armed", "elapsed", "start_sample"):
        assert np.array_equal(d1[k][~touched], d0[k][~touched]), k


# ---- launches and refusals ---------------------------------------------------------------------------------------------------------------
def _same_state(a, b):
    return all(np.array_equal(np.asarray(a[k]).view(np.uint8) if isinstance(a[k], np.ndarray) else a[k],
                              np.asarray(b[k]).view(np.uint8) if isinstance(b[k], np.ndarray) else b[k]) for k in a)


def test_one_launch_each_and_refusals_leave_everything_unchanged():
    import torch
    from microwakeword_b200 import _lib
    from microwakeword_b200.endpoint import Endpointer
    from microwakeword_b200.engine import StreamEngine
    S = 65536
    eng = StreamEngine(F32, n_streams=S)
    eng.set_audio_history(480)
    ep = Endpointer(eng, **RULE)
    bank = _audio_bank(13, 16000, 5)
    for c in range(6):
        ep.update(torch.rand((S, eng.step(_streams_audio(bank, S, c)).shape[1]), device="cuda"))
    ep.arm(np.arange(0, S, 3))
    for n in (1, S):
        ids = np.random.default_rng(n).permutation(S)[:n]
        L0 = ep.launch_count
        recs = ep.export_streams(ids)
        assert ep.launch_count - L0 == 1
        ep.import_streams(ids, recs)
        assert ep.launch_count - L0 == 2
    L, st = ep._L, _stream()
    recs = ep.export_streams(np.arange(4))
    ids4 = np.arange(4, dtype=np.int32)
    torch.cuda.synchronize()
    state, launches = ep.state_dict(), ep.launch_count

    def refused(rc, word=None):
        assert rc == -1                                              # MWW_EINVAL
        msg = L.mww_last_error(None).decode()
        assert word is None or word in msg, msg

    for field, v in (("vad_window", 4), ("stride", 1), ("hop_samples", 320), ("buffered", 0), ("pending", 2), ("record_bytes", 96)):
        lay = _lib.MwwEndpointerLayout.from_buffer_copy(recs.layout)
        setattr(lay, field, v)
        refused(L.mww_import_endpointer_rows(ep._ep, ids4.ctypes.data, 4, recs.data.data_ptr(), ctypes.byref(lay), st), field)
    refused(L.mww_import_endpointer_rows(ep._ep, ids4.ctypes.data, -1, recs.data.data_ptr(), ctypes.byref(recs.layout), st))
    refused(L.mww_import_endpointer_rows(ep._ep, ids4.ctypes.data, 4, recs.data.data_ptr(), None, st), "layout")
    refused(L.mww_import_endpointer_rows(ep._ep, ids4.ctypes.data, 4, None, ctypes.byref(recs.layout), st))
    refused(L.mww_import_endpointer_rows(ep._ep, ids4.ctypes.data, 1, recs.data.data_ptr() + 4, ctypes.byref(recs.layout), st), "aligned")
    refused(L.mww_export_endpointer_rows(ep._ep, ids4.ctypes.data, 1, recs.data.data_ptr() + 8, None, st), "aligned")
    for bad in ([0, 0, 1, 2], [0, 1, 2, S]):
        b = np.asarray(bad, np.int32)
        refused(L.mww_import_endpointer_rows(ep._ep, b.ctypes.data, 4, recs.data.data_ptr(), ctypes.byref(recs.layout), st))
    b = np.asarray([-1], np.int32)
    refused(L.mww_export_endpointer_rows(ep._ep, b.ctypes.data, 1, recs.data.data_ptr(), None, st), "out of range")
    # behind the handle: a call without ep.update
    eng.step(_streams_audio(bank, S, 9))
    refused(L.mww_export_endpointer_rows(ep._ep, ids4.ctypes.data, 4, recs.data.data_ptr(), None, st),
            "update the endpointer after the handle's last call")
    refused(L.mww_import_endpointer_rows(ep._ep, ids4.ctypes.data, 4, recs.data.data_ptr(), ctypes.byref(recs.layout), st),
            "update the endpointer after the handle's last call")
    torch.cuda.synchronize()
    assert ep.launch_count == launches and _same_state(ep.state_dict(), state)
    # the history write's refusals leave the history and the launch count as they were
    hist, hl = eng.audio_history(np.arange(S), 480).clone(), eng.launch_count
    rows = torch.ones((4, 480), dtype=torch.int16, device="cuda")
    for rc in (_write(eng, [0, 0, 1, 2], rows), _write(eng, [0, 1, 2, S], rows), _write(eng, [0, 1, 2, 3], rows, stride=479),
               _write(eng, [0, 1, 2, 3], rows, n_samples=(1 << 22) + 8, stride=1 << 23), _write(eng, [0, 1, 2, 3], rows, ptr=0),
               _write(eng, [0, 1, 2, 3], rows, n_samples=-1)):
        assert rc != 0
    plain = StreamEngine(F32, n_streams=8)
    assert _write(plain, [0], rows[:1]) != 0 and b"no audio history" in plain._L.mww_last_error(plain._h)
    assert eng.launch_count == hl and torch.equal(eng.audio_history(np.arange(S), 480), hist)
