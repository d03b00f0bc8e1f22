"""Endpointing (mww_endpointer_*; microwakeword_b200.endpoint.Endpointer), the parts that need no GPU: the kernels' per-row
bodies (microwakeword_b200/csrc/mww_endpoint.h, built with g++ in a temporary directory by tests/emul_endpoint.cc), driven
as the C-ABI drives them, against tests/endpoint_ref.py, a NumPy model written from the rule in include/mww.h -- random VAD
tracks split into calls anywhere, every end reason and the ties between them, re-arm, disarm and reset between calls, the
lookback replay, the speech flag against tests/detector_models_ref.py's VAD, the position formula against a replay of the
frontend's row counting, and the command read's slot math -- and the refusals, the symbols, the companion library and the
timing tool's loud failure without a GPU."""

import ctypes
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import endpoint_ref as R
from conftest import GOLDEN, ROOT
from detector_models_ref import VAD, WAKE, ModelsRef

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_endpoint_test_")
_emul = None


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_endpoint.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_endpoint.cc")], check=True)
        _emul = ctypes.CDLL(so)
        vp, i32, ll, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_double
        _emul.emul_endpoint_update.argtypes = [vp, d, ll, vp, vp, ll, i32, ll]
        _emul.emul_endpoint_arm.argtypes = [vp, d, ll, vp, vp, i32, i32, i32, vp]
        _emul.emul_endpoint_clear.argtypes = [vp, d, ll, vp, vp, i32, i32]
        _emul.emul_endpoint_position.argtypes = [ll, i32, i32, i32, i32, i32, i32]
        _emul.emul_endpoint_position.restype = ll
        _emul.emul_endpoint_fits.argtypes = [ll, i32, i32, ll, i32, i32, i32, i32, i32]
        _emul.emul_endpoint_fits.restype = i32
        _emul.emul_endpoint_read.argtypes = [vp, i32, ll, ll, vp, i32, ll, ll, i32, vp, ll, vp]
        for f in (_emul.emul_endpoint_update, _emul.emul_endpoint_arm, _emul.emul_endpoint_clear, _emul.emul_endpoint_read):
            f.restype = None
    return _emul


class Emul:
    """the C-ABI's host logic (mww_endpoint_capi.cu) over the header's bodies: state arrays, the baseline counters, the
    consistency check, the position ring and the arm tags"""

    def __init__(self, n_streams, members, stride, hop, vad_window=5, vad_cutoff=0.5, speech_steps=3, silence_steps=25, timeout_steps=100,
                 max_steps=334, lookback_steps=64, capacity=64, counters=(0, 0, 0)):
        self.members = np.asarray(members, np.int32)
        Rn = self.members.size
        self.stride, self.hop, self.capacity, self.w, self.lookback = stride, hop, capacity, vad_window, lookback_steps
        self.cfg = np.array([vad_window, speech_steps, silence_steps, timeout_steps, max_steps, lookback_steps, Rn, n_streams, capacity], np.int32)
        self.cutoff, self.step_samples = float(vad_cutoff), stride * hop
        self.row_of = np.full(n_streams, -1, np.int32)
        self.row_of[self.members] = np.arange(Rn)
        self.a = dict(hist=np.zeros((max(vad_window - 1, 0), Rn), np.float32), seen=np.zeros(Rn, np.int64), flags=np.zeros(Rn, np.uint64),
                      armed=np.full(Rn, -1, np.int32), elapsed=np.zeros(Rn, np.int32), run=np.zeros(Rn, np.int32),
                      silence=np.zeros(Rn, np.int32), heard=np.zeros(Rn, np.int32), start=np.zeros(Rn, np.int64),
                      speech_end=np.zeros(Rn, np.int64), arm_tag=np.zeros(Rn, np.int32), row_of=self.row_of,
                      count=np.zeros(1, np.uint64), events=np.zeros(capacity, R.EVENT), ended=np.full(capacity, -1, np.int32))
        order = ("hist", "seen", "flags", "armed", "elapsed", "run", "silence", "heard", "start", "speech_end", "arm_tag", "row_of", "count",
                 "events", "ended")
        self.ptrs = (ctypes.c_void_p * 15)(*[self.a[k].ctypes.data for k in order])
        self.base, self.steps, self.pos, self.tag = tuple(counters), 0, np.zeros(64, np.int64), 0

    def _c(self):
        return self.cfg.ctypes.data, self.cutoff, self.step_samples, self.ptrs

    def update(self, probs, S, buffered, pending):
        probs = np.ascontiguousarray(probs, np.float32)
        n = probs.shape[1]
        if not emul().emul_endpoint_fits(self.base[0], self.base[1], self.base[2], S, buffered, pending, self.hop, self.stride, n):
            raise ValueError("inconsistent update")
        pos0 = emul().emul_endpoint_position(S, buffered, self.hop, pending, self.stride, n, 0)
        emul().emul_endpoint_update(*self._c(), probs.ctypes.data, n, n, pos0)
        self.base = (S, buffered, pending)
        keep = min(n, 64)
        self.pos[keep:] = self.pos[:64 - keep].copy()
        self.pos[:keep] = pos0 + (n - 1 - np.arange(keep)) * self.step_samples
        self.steps += n

    def arm(self, ids):
        ids = np.ascontiguousarray(ids, np.int32)
        self.tag += 1
        emul().emul_endpoint_arm(*self._c(), ids.ctypes.data, ids.size, min(self.lookback, self.steps), self.tag, self.pos.ctypes.data)

    def clear(self, ids, reset, counters=None):
        if ids is None:
            emul().emul_endpoint_clear(*self._c(), None, self.members.size, reset)
            self.base, self.steps, self.pos = tuple(counters), 0, np.zeros(64, np.int64)
        else:
            ids = np.ascontiguousarray(ids, np.int32)
            emul().emul_endpoint_clear(*self._c(), ids.ctypes.data, ids.size, reset)

    def drain(self):
        n = int(self.a["count"][0])
        ev = self.a["events"][:min(n, self.capacity)].copy()
        self.a["count"][0] = 0
        self.a["ended"][:] = -1
        return ev, n

    def state(self):
        a = self.a
        return dict(hist=a["hist"].T.copy(), seen=a["seen"].copy(), flags=a["flags"].copy(), armed=a["armed"].copy(), elapsed=a["elapsed"].copy(),
                    run=a["run"].copy(), silence=a["silence"].copy(), heard=a["heard"].copy(), start_sample=a["start"].copy(),
                    speech_end_sample=a["speech_end"].copy(), samples_seen=self.base[0], buffered=self.base[1], pending=self.base[2],
                    steps=self.steps, positions=self.pos.copy())


def sort_events(ev):
    ev = np.asarray(ev, R.EVENT)
    return ev[np.lexsort((ev["stream"], ev["end_sample"]))]


def same_state(a, b):
    for k in ("hist", "seen", "flags", "armed", "elapsed", "run", "silence", "heard", "start_sample", "speech_end_sample", "positions"):
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.shape != y.shape or not np.array_equal(x.astype(np.float64 if k == "hist" else np.int64) if k != "flags" else x.astype(np.uint64),
                                                    y.astype(np.float64 if k == "hist" else np.int64) if k != "flags" else y.astype(np.uint64)):
            return False
    return all(int(a[k]) == int(b[k]) for k in ("samples_seen", "buffered", "pending", "steps"))


class Frontend:
    """the handle's lockstep counters: buffered samples, the model's pending rows and samples_seen of the history"""

    def __init__(self, hop=160, stride=3, seen=0, buffered=0):
        self.hop, self.stride, self.buffered, self.pending, self.S = hop, stride, buffered, 0, seen
        self.row_ends = []                                   # position of every row's last sample

    def call(self, n16):
        rows = (self.buffered + n16 - 480) // self.hop + 1 if self.buffered + n16 >= 480 else 0
        for r in range(rows):                                # the window of a row ends 480 - buffered samples into the call, then each hop
            self.row_ends.append(self.S + (480 - self.buffered) + r * self.hop)
        steps = (self.pending + rows) // self.stride
        step_ends = [self.row_ends[len(self.row_ends) - rows - self.pending + (j + 1) * self.stride - 1] for j in range(steps)]
        self.pending = (self.pending + rows) % self.stride
        self.buffered = self.buffered + n16 - rows * self.hop
        self.S += n16
        return steps, step_ends

    def counters(self):
        return self.S, self.buffered, self.pending


def _tracks(rng, R_, n):
    """speech-like probabilities: runs of high and low values, some rows noisy"""
    out = np.empty((R_, n), np.float32)
    for r in range(R_):
        level = rng.random() < 0.5
        j = 0
        while j < n:
            L = int(rng.integers(1, 30))
            out[r, j:j + L] = np.clip((0.85 if level else 0.1) + rng.normal(0, 0.25, min(L, n - j)), 0, 1)
            level = not level
            j += L
    return out


RULE = dict(vad_window=5, vad_cutoff=0.5, speech_steps=3, silence_steps=6, timeout_steps=20, max_steps=45, lookback_steps=10, capacity=64)


def _steps_of(fe, n16):
    """the steps a call of n16 samples would give, without making it"""
    rows = (fe.buffered + n16 - 480) // fe.hop + 1 if fe.buffered + n16 >= 480 else 0
    return (fe.pending + rows) // fe.stride


def _drive_exact(obj, fe, probs, ops, splits, rng):
    """feed obj the steps of probs through calls drawn from splits, never past the next step count that has ops: a call that
    would go past it is replaced by calls of hop samples, which give at most one row each.  At each step count in ops the same
    operations run, so every split sees them between the same steps.  -> the drains, in order."""
    total, used, drains = probs.shape[1], 0, []
    stops = sorted(set(ops) | {total})
    for stop in stops:
        while used < stop:
            n16 = int(rng.choice(splits))
            if used + _steps_of(fe, n16) > stop:
                n16 = fe.hop
            steps, _ = fe.call(n16)
            obj.update(probs[:, used:used + steps], *fe.counters())
            used += steps
        for op, ids in ops.get(stop, []):
            if op == "drain":
                drains.append(obj.drain())
            elif isinstance(obj, R.EndpointRef):
                getattr(obj, op)(ids)
            else:
                {"arm": obj.arm, "disarm": lambda i: obj.clear(i, 0), "reset": lambda i: obj.clear(i, 1)}[op](ids)
    drains.append(obj.drain())
    return drains


SPLITS = {"live": [480], "mixed": [480, 480, 480, 160, 1000, 37, 4800, 0], "long": [3360, 13, 9999]}


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("stride,hop", [(3, 160), (1, 160), (2, 320), (5, 96)])
def test_random_tracks_match_the_reference_however_split(seed, stride, hop):
    """the same probabilities and the same operations between the same steps, through three different splits into calls:
    every split gives the reference's events and state, bit for bit.  With a capacity that overflows, the true counts still
    agree and the kept events are some of those events: which ones depends on the order within a call, which is unspecified."""
    rng = np.random.default_rng(seed * 31 + stride)
    n_streams, total = 24, 300
    members = np.sort(rng.choice(n_streams, 17, replace=False)).astype(np.int32)
    lookback = int(rng.choice([0, 1, 10, 64]))
    probs = _tracks(rng, members.size, total)
    ops = {}
    for at in sorted(rng.choice(np.arange(1, total), 40, replace=False).tolist()):
        kind = rng.choice(["arm", "arm", "arm", "disarm", "reset", "drain"])
        ids = rng.integers(-2, n_streams + 2, 6).astype(np.int32) if kind == "arm" else rng.integers(0, n_streams, 2).astype(np.int32)
        if kind == "arm":
            ids = np.concatenate([ids, ids[:2]])                        # repeats arm once
        ops.setdefault(int(at), []).append((str(kind), ids))
    ops.setdefault(0, []).append(("arm", members))
    runs = {}
    for capacity in (256, 4):
        for name, splits in SPLITS.items():
            for kind in ("ref", "emul"):
                fe = Frontend(hop, stride, seen=1000)
                cls = R.EndpointRef if kind == "ref" else Emul
                obj = cls(n_streams, members, stride, hop, counters=fe.counters(), **dict(RULE, lookback_steps=lookback, capacity=capacity))
                drains = _drive_exact(obj, fe, probs, ops, splits, np.random.default_rng(seed))
                runs[capacity, name, kind] = ([sort_events(d[0]) for d in drains], [d[1] for d in drains], obj.state())
    base_events, base_counts, base_state = runs[256, "live", "ref"]
    assert sum(base_counts) == sum(e.size for e in base_events) > 0                 # nothing dropped at this capacity
    for (capacity, name, kind), (events, counts, state) in runs.items():
        key = (capacity, name, kind)
        assert counts == base_counts, key
        if capacity == 256:
            assert all(np.array_equal(a, b) for a, b in zip(events, base_events)), key
        else:
            assert all(e.size == min(c, capacity) and np.isin(e, b).all() for e, c, b in zip(events, counts, base_events)), key
        assert state["steps"] == total
        same = dict(state, samples_seen=base_state["samples_seen"], buffered=base_state["buffered"], pending=base_state["pending"])
        assert same_state(same, base_state), key                                    # every row field, the flags and the positions
        assert same_state(state, runs[capacity, name, "ref"][2]), key               # within one split, the counters too
    assert sum(runs[4, "live", "ref"][1]) > sum(e.size for e in runs[4, "live", "ref"][0])      # the small capacity dropped some


def _one_row(flags, lookback=0, arm_at=0, **kw):
    """one stream fed the flags (1.0 / 0.0 with window 1), armed before step arm_at -> (ref, emul) after the steps"""
    rule = dict(RULE, vad_window=1, lookback_steps=lookback)
    rule.update(kw)
    fe = Frontend(buffered=320)                             # steady live calls: one step per 480 samples, ending at 480 (j + 1)
    objs = [R.EndpointRef(1, [0], 3, 160, counters=fe.counters(), **rule), Emul(1, [0], 3, 160, counters=fe.counters(), **rule)]
    for j, f in enumerate(flags):
        if j == arm_at:
            for o in objs:
                o.arm([0])
        steps, _ = fe.call(480)
        for o in objs:
            o.update(np.array([[1.0 if f else 0.0]], np.float32), *fe.counters())
    if arm_at >= len(flags):
        for o in objs:
            o.arm([0])
    return objs


@pytest.mark.parametrize("flags,reason,steps", [
    ([1, 1, 1, 0, 0, 0, 0, 0, 0], R.END_OF_SPEECH, 9),
    ([0] * 20, R.NO_SPEECH, 20),
    ([1, 1, 1] + [1, 0] * 30, R.MAX_LENGTH, 45),     # heard, and never 6 silent steps in a row
])
def test_every_end_reason(flags, reason, steps):
    kw = dict(timeout_steps=100) if reason == R.MAX_LENGTH else {}
    ref, em = _one_row(flags, **kw)
    (er, nr), (ee, ne) = ref.drain(), em.drain()
    assert nr == ne == 1 and np.array_equal(sort_events(er), sort_events(ee))
    assert er["reason"][0] == reason and er["steps"][0] == steps
    e = er[0]
    assert e["start_sample"] == 480 - 480 and e["end_sample"] == 480 * steps     # step j of 480-sample live calls ends at 480 (j + 1)
    if reason == R.END_OF_SPEECH:
        assert e["speech_end_sample"] == 480 * 3
    elif reason == R.NO_SPEECH:
        assert e["speech_end_sample"] == e["start_sample"]
    else:
        assert e["speech_end_sample"] == 480 * 44                # the last speech step before the end


def test_ties_on_one_step_go_in_rule_order():
    # END_OF_SPEECH and MAX_LENGTH on the same step
    ref, em = _one_row([1, 1, 1, 0, 0, 0], silence_steps=3, max_steps=6)
    (er, _), (ee, _) = ref.drain(), em.drain()
    assert er["reason"].tolist() == ee["reason"].tolist() == [R.END_OF_SPEECH]
    # NO_SPEECH and MAX_LENGTH on the same step
    ref, em = _one_row([0] * 5, timeout_steps=5, max_steps=5)
    (er, _), (ee, _) = ref.drain(), em.drain()
    assert er["reason"].tolist() == ee["reason"].tolist() == [R.NO_SPEECH]
    # heard on the step that reaches the timeout: not NO_SPEECH
    ref, em = _one_row([0, 1, 1, 1], speech_steps=3, timeout_steps=4, max_steps=4)
    (er, _), (ee, _) = ref.drain(), em.drain()
    assert er["reason"].tolist() == ee["reason"].tolist() == [R.MAX_LENGTH]


@pytest.mark.parametrize("lookback", [0, 1, 10, 64])
def test_lookback_is_arming_earlier(lookback):
    """arm_at below the lookback: every step consumed since create is replayed"""
    rng = np.random.default_rng(lookback)
    flags = (rng.random(120) < 0.5).tolist()
    L = lookback
    for arm_at in (0, 3, 50, 119, 120):
        late = _one_row(flags, lookback=lookback, arm_at=arm_at, timeout_steps=1000, max_steps=1000, silence_steps=1000)
        early = _one_row(flags, lookback=0, arm_at=max(arm_at - min(L, arm_at), 0), timeout_steps=1000, max_steps=1000, silence_steps=1000)
        for a, b in zip(late, early):
            sa, sb = a.state(), b.state()
            for k in R.SEG if isinstance(a, R.EndpointRef) else ("elapsed", "run", "silence", "heard", "start_sample", "speech_end_sample"):
                assert int(sa[k][0]) == int(sb[k][0]), (k, arm_at)
        assert int(late[0].state()["elapsed"][0]) == min(L, arm_at) + (120 - arm_at)


def test_replay_reaches_an_end_during_arm_and_more_than_steps_consumed():
    ref, em = _one_row([0] * 30, lookback=64, arm_at=30, timeout_steps=20)
    (er, _), (ee, _) = ref.drain(), em.drain()
    assert er["reason"].tolist() == ee["reason"].tolist() == [R.NO_SPEECH] and er["end_sample"][0] == ee["end_sample"][0] == 480 * 20
    assert ref.state()["armed"][0] == em.state()["armed"][0] == -1
    ref, em = _one_row([1] * 5, lookback=64, arm_at=5)                # L = min(64, 5)
    assert int(ref.state()["elapsed"][0]) == int(em.state()["elapsed"][0]) == 5


def test_no_replay_reaches_across_a_whole_reset():
    """a whole reset takes a new baseline, which may start a new axis: the steps and positions before it are forgotten"""
    for o in _one_row([1, 1, 1, 1, 0, 0], lookback=64, arm_at=99):
        o_state = o.state()
        assert o_state["steps"] == 6 and o_state["positions"][0] == 480 * 6
        if isinstance(o, R.EndpointRef):
            o.reset(None, counters=(0, 320, 0))
        else:
            o.clear(None, 1, counters=(0, 320, 0))
        o.arm([0])
        st = o.state()
        assert st["steps"] == 0 and not st["positions"].any() and int(st["elapsed"][0]) == 0 and int(st["armed"][0]) == 0
        o.update(np.array([[1.0]], np.float32), 480, 320, 0)          # the new axis: the first step ends at 480
        st = o.state()
        assert int(st["start_sample"][0]) == 0 and int(st["elapsed"][0]) == 1


def test_rearm_disarm_reset_between_calls():
    fe = Frontend(buffered=320)
    objs = [R.EndpointRef(4, [0, 1, 2, 3], 3, 160, counters=fe.counters(), **RULE), Emul(4, [0, 1, 2, 3], 3, 160, counters=fe.counters(), **RULE)]
    rng = np.random.default_rng(4)
    probs = _tracks(rng, 4, 100)
    for j in range(100):
        fe.call(480)
        for o in objs:
            o.update(probs[:, j:j + 1], *fe.counters())
            if j == 10:
                o.arm([0, 1, 2, 3])
            if j == 14:
                o.arm([1])                                          # re-arm restarts
            if j == 16:
                (o.disarm if isinstance(o, R.EndpointRef) else (lambda i: o.clear(i, 0)))([2])
            if j == 18:
                (o.reset if isinstance(o, R.EndpointRef) else (lambda i: o.clear(i, 1)))([3])
    assert same_state(objs[0].state(), objs[1].state())
    (er, _), (ee, _) = objs[0].drain(), objs[1].drain()
    assert np.array_equal(sort_events(er), sort_events(ee))
    assert 2 not in er["stream"].tolist()


def test_speech_flags_equal_the_models_detector_vad():
    rng = np.random.default_rng(7)
    for w, cutoff in ((1, 0.5), (5, 0.5), (32, 0.3)):
        n_streams, members = 9, np.array([1, 4, 5, 8], np.int32)
        md = ModelsRef(n_streams, [WAKE, VAD], [5, w], [0.99, cutoff], [0, 0], [3, 3], streams=[None, members])
        fe = Frontend(buffered=320)
        em = Emul(n_streams, members, 3, 160, vad_window=w, vad_cutoff=cutoff, counters=fe.counters())
        probs = _tracks(rng, members.size, 120)
        probs[0, 7] = np.nan
        for j in range(120):
            fe.call(480)
            em.update(probs[:, j:j + 1], *fe.counters())
            md.update([np.zeros((n_streams, 1), np.float32), probs[:, j:j + 1]], [1, 1], [0, 0])
            assert np.array_equal(em.state()["flags"] & np.uint64(1), md.flag[1].astype(np.uint64)), j


@pytest.mark.parametrize("stride", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("hop", [160, 320, 96, 480])
def test_position_formula_against_the_frontends_row_counting(stride, hop):
    rng = np.random.default_rng(stride * 1000 + hop)
    fe = Frontend(hop, stride, seen=int(rng.integers(0, 10 ** 6)))
    base = fe.counters()
    pendings = set()
    for _ in range(200):
        n16 = int(rng.choice([480, 480, 1, 159, 160, 161, 4000, 16000, 0, 7]))
        steps, ends = fe.call(n16)
        S, b, g = fe.counters()
        pendings.add(g)
        assert emul().emul_endpoint_fits(*base, S, b, g, hop, stride, steps)
        assert not emul().emul_endpoint_fits(*base, S, b, g, hop, stride, steps + 1)
        if steps:
            assert not emul().emul_endpoint_fits(*base, S, b, g, hop, stride, steps - 1)
        got = [emul().emul_endpoint_position(S, b, hop, g, stride, steps, j) for j in range(steps)]
        assert got == ends == [R.position(S, b, hop, g, stride, steps, j) for j in range(steps)]
        base = (S, b, g)
    assert pendings == set(range(stride)) or stride == 1


def test_live_calls_have_b_zero():
    fe = Frontend(160, 3)
    for _ in range(10):
        fe.call(480)
        assert fe.buffered - (480 - 160) == 0


def _read(ring, C, seen, events, count, capacity, pre, post, max_samples, out_stride=None):
    out_stride = out_stride or max(max_samples, 1)
    out = np.full((capacity, out_stride), 12345, np.int16)
    lengths = np.full(capacity, -7, np.int32)
    ev = np.ascontiguousarray(events, R.EVENT)
    emul().emul_endpoint_read(np.ascontiguousarray(ring).ctypes.data, C, seen, count, ev.ctypes.data, capacity, pre, post, max_samples,
                              out.ctypes.data, out_stride, lengths.ctypes.data)
    return out[:, :max_samples], lengths


@pytest.mark.parametrize("C,seen", [(64, 40), (64, 64), (64, 1000), (800, 5000)])
@pytest.mark.parametrize("count", [0, 3, 8, 20])
def test_command_read_slot_math(C, seen, count):
    rng = np.random.default_rng(C + seen + count)
    n_streams, capacity = 5, 8
    # the ring as the history writes it: sample t of stream s at slot t mod C, for t in [seen - C, seen)
    truth = rng.integers(-30000, 30000, (n_streams, seen + 10)).astype(np.int16)
    ring = np.zeros((n_streams, C), np.int16)
    for t in range(max(0, seen - C), seen):
        ring[:, t % C] = truth[:, t]
    ev = np.zeros(capacity, R.EVENT)
    ev["stream"] = rng.integers(0, n_streams, capacity)
    ev["reason"] = rng.integers(1, 4, capacity)
    ev["start_sample"] = rng.integers(seen - 2 * C, seen, capacity)
    ev["speech_end_sample"] = ev["start_sample"] + rng.integers(0, C, capacity)
    ev["end_sample"] = ev["speech_end_sample"] + rng.integers(1, C, capacity)
    ev["end_sample"][0] = seen + 20                                        # reaches past samples_seen
    for pre, post, max_samples in ((0, 0, C), (16, 24, 2 * C), (5, 3, 7), (0, 0, 0)):
        got, lengths = _read(ring, C, seen, ev, count, capacity, pre, post, max_samples)

        def last_C(s):
            return np.array([truth[s, t] if t >= 0 else 0 for t in range(seen - C, seen)], np.int16)

        want, wl = R.commands(ev, count, capacity, pre, post, max_samples, seen, C, last_C)
        assert np.array_equal(lengths, wl) and np.array_equal(got, want)
        assert (lengths[min(count, capacity):] == 0).all() and (lengths <= max_samples).all()


def test_command_span_truncates_keeping_the_beginning():
    e = np.zeros(1, R.EVENT)
    e["reason"], e["start_sample"], e["speech_end_sample"], e["end_sample"] = R.END_OF_SPEECH, 1000, 5000, 9000
    assert R.command_span(e[0], 100, 200, 10 ** 6) == (900, 5200 - 900)
    assert R.command_span(e[0], 100, 10 ** 6, 10 ** 6) == (900, 9000 - 900)
    assert R.command_span(e[0], 100, 200, 50) == (900, 50)
    e["reason"] = R.MAX_LENGTH
    assert R.command_span(e[0], 0, 200, 10 ** 6) == (1000, 8000)


# ---- ABI ------------------------------------------------------------------------------------------------------------------------------
NEW = ("mww_endpointer_create", "mww_endpointer_destroy", "mww_endpointer_info", "mww_endpointer_update", "mww_endpointer_arm",
       "mww_endpointer_arm_device", "mww_endpointer_disarm", "mww_endpointer_reset", "mww_endpointer_reset_device", "mww_endpointer_drain",
       "mww_endpointer_buffers", "mww_endpointer_get_state", "mww_endpointer_set_state", "mww_endpointer_read_commands")


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    assert all(n in _lib.EXPORTS and hasattr(L, n) for n in NEW)
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    assert all(re.search(r"\bT %s\b" % n, syms) for n in NEW)
    hdr = open(os.path.join(ROOT, "include", "mww.h")).read()
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S))
    assert "int mww_endpointer_create(const mww_t *h, int model, const mww_endpoint_rule *rule, int capacity, mww_endpointer_t **out);" in flat
    assert "int mww_endpointer_update(mww_endpointer_t *ep, const float *d_probs, int n, long long pitch, void *cu_stream);" in flat
    assert ("int mww_endpointer_read_commands(mww_endpointer_t *ep, mww_t *h, long long pre, long long post, int max_samples, int16_t *d_out, "
            "long long out_stride, int32_t *d_lengths, void *cu_stream);") in flat
    assert ("typedef struct mww_endpoint_event { int32_t stream, reason; int64_t start_sample, end_sample, speech_end_sample; "
            "int32_t steps, pad; } mww_endpoint_event;") in flat
    assert ctypes.sizeof(_lib.MwwEndpointEvent) == 40 == R.EVENT.itemsize
    assert ctypes.sizeof(_lib.MwwEndpointRule) == 32 and ctypes.sizeof(_lib.MwwEndpointerDesc) == 24 + 32 + 16
    assert ctypes.sizeof(_lib.MwwEndpointState) == 10 * 8 + 4 * 8 + 64 * 8
    vp, i32, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    assert L.mww_endpointer_update.argtypes == [vp, vp, i32, ll, vp]
    assert L.mww_endpointer_read_commands.argtypes == [vp, vp, ll, ll, i32, vp, ll, vp, vp]


def _rule(**kw):
    from microwakeword_b200 import _lib
    r = dict(vad_window=5, speech_steps=3, silence_steps=25, timeout_steps=100, max_steps=334, lookback_steps=64, vad_cutoff=0.5)
    r.update(kw)
    return _lib.MwwEndpointRule(r["vad_window"], r["speech_steps"], r["silence_steps"], r["timeout_steps"], r["max_steps"], r["lookback_steps"],
                                r["vad_cutoff"])


def test_c_refusals_before_any_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    out = ctypes.c_void_p(1)
    assert L.mww_endpointer_create(None, 0, ctypes.byref(_rule()), 4, ctypes.byref(out)) == -1 and out.value is None
    assert b"handle" in L.mww_last_error(None)
    assert L.mww_endpointer_info(None, None) == -1
    for name in ("mww_endpointer_arm", "mww_endpointer_arm_device", "mww_endpointer_disarm", "mww_endpointer_reset", "mww_endpointer_reset_device"):
        assert getattr(L, name)(None, None, 0, None) == -1 and b"endpointer" in L.mww_last_error(None)
    assert L.mww_endpointer_update(None, None, 0, 0, None) == -1
    assert L.mww_endpointer_drain(None, None, 0, None, None) == -1
    assert L.mww_endpointer_read_commands(None, None, 0, 0, 0, None, 0, None, None) == -1
    assert L.mww_endpointer_get_state(None, None) == -1 and L.mww_endpointer_set_state(None, None) == -1
    assert L.mww_endpointer_destroy(None) == 0


class NoLib:
    def __getattr__(self, name):
        raise AssertionError("the library was called: %s" % name)


def test_python_refusals_before_the_library_is_called(monkeypatch):
    from microwakeword_b200 import _lib
    from microwakeword_b200.endpoint import Endpointer

    def no_lib():
        raise AssertionError("the library was loaded")

    monkeypatch.setattr(_lib, "lib", no_lib)

    class Eng:
        _h, device, n_streams, audio_history_capacity = ctypes.c_void_p(1), 0, 8, 1600

    for kw in (dict(vad_window=0), dict(vad_window=33), dict(vad_cutoff=float("nan")), dict(vad_cutoff="0.5"), dict(speech_steps=0),
               dict(silence_steps=0), dict(timeout_steps=0), dict(max_steps=0), dict(lookback_steps=-1), dict(lookback_steps=65),
               dict(capacity=0), dict(capacity=1.5), dict(model=1), dict(model=-1), dict(model=True)):
        with pytest.raises(ValueError):
            Endpointer(Eng(), **kw)
    eng = Eng()
    eng.audio_history_capacity = 0
    with pytest.raises(ValueError):
        Endpointer(eng)
    with pytest.raises(ValueError):
        Endpointer(object())
    ep = object.__new__(Endpointer)
    ep.__dict__.update(_L=NoLib(), device=0, capacity=8, n_rows=4, engine=Eng())
    for kw in (dict(pre=-1), dict(post=-1), dict(max_samples=-1), dict(max_samples=(1 << 22) + 1), dict(pre=0.5)):
        with pytest.raises(ValueError):
            ep.commands(**kw)
    for bad in ([8], [-1], [0.5], [[0, 1]]):
        with pytest.raises(ValueError):
            ep.arm(bad)
    with pytest.raises(ValueError):
        ep.update(np.zeros((4, 1), np.float32))


# ---- build ----------------------------------------------------------------------------------------------------------------------------
def _res_usage(so):
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return subprocess.run([tool, "-res-usage", so], capture_output=True, text=True, check=True).stdout


def test_companion_library_holds_exactly_its_four_kernels_without_stack_or_local_memory():
    from microwakeword_b200 import build
    assert os.path.basename(build.EP_OUT) == "libmww_endpoint.so" and build.EP_SOURCES == ["mww_endpoint.cu"]
    assert "mww_endpoint_capi.cu" in build.SOURCES and "mww_endpoint.cu" not in build.SOURCES
    res = _res_usage(build.EP_OUT)
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    names = sorted(n for n, *_ in found)
    assert len(names) == 4, res
    for k in ("endpoint_update_kernel", "endpoint_arm_kernel", "endpoint_clear_kernel", "endpoint_read_kernel"):
        assert any(k in n for n in names), (k, res)
    assert all(int(stack) == int(local) == 0 for _, _, stack, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "endpoint.cubin"),
                                                 os.path.join(CSRC, "mww_endpoint.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 4 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    main = _res_usage(build.OUT)
    assert not any(k in main for k in ("endpoint_update_kernel", "endpoint_arm_kernel", "endpoint_clear_kernel", "endpoint_read_kernel"))
    if shutil.which("readelf"):
        dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True, check=True).stdout
        assert "[libmww_endpoint.so]" in dyn and "$ORIGIN" in dyn


def test_stale_check_covers_the_companion_library(monkeypatch):
    from microwakeword_b200 import build
    real = os.path.exists
    monkeypatch.setattr(os.path, "exists", lambda p: False if p == build.EP_OUT else real(p))
    assert build._stale()


def test_timing_tool_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(ROOT, "tools", "endpoint_time.py")
    res = subprocess.run([sys.executable, tool, "--rounds", "1"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
