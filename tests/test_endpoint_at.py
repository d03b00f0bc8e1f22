"""The positioned arm of the endpointer (mww_endpointer_arm_at, include/mww.h "positioned arm"; Endpointer.arm(ids, at=...)),
the parts that need no GPU: the positioned per-row bodies of microwakeword_b200/csrc/mww_endpoint.h and mww_serving_records.h,
built with g++ by tests/emul_endpoint_at.cc and driven as the C-ABI drives them, against tests/endpoint_at_ref.py, the NumPy
statement of the rule -- positions on and between grid points, in the future, older than the replay and negative; skip 0 and
mutes over several updates; run-on speech inside the skip, an end during the replay, re-arming, disarm and reset mid-mute,
duplicate ids, no steps after a whole reset; the rule's three properties; records with and without mute words -- and the
symbols, the Python refusals, the new library's kernels and resources, and every existing library's instructions against
tests/golden/sass_kernels_before_endpoint_at.json (the parent's build)."""

import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import endpoint_ref as R
from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import endpoint_at_ref as A  # noqa: E402
import test_endpoint as TE  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_endpoint_at_test_")
_emul = []
vp, i32, ll, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_double


def emul():
    if not _emul:
        so = os.path.join(_BUILD.name, "libemul_endpoint_at.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", HERE, "-o", so, os.path.join(HERE, "emul_endpoint_at.cc")],
                       check=True)
        L = ctypes.CDLL(so)
        L.emul_at_update.argtypes = [vp, d, ll, vp, vp, vp, ll, i32, ll]
        L.emul_at_arm.argtypes = [vp, d, ll, vp, vp, vp, i32, i32, i32, vp]
        L.emul_at_clear.argtypes = [vp, d, ll, vp, vp, vp, i32, i32]
        L.emul_at_arm_at.argtypes = [vp, d, ll, vp, vp, vp, vp, vp, i32, vp, i32, i32, vp, ll, ll]
        L.emul_at_record_bytes.argtypes = [i32]
        L.emul_at_record_bytes.restype = ll
        L.emul_at_pack.argtypes = [vp, d, ll, vp, vp, ll, vp, i32, vp, i32]
        L.emul_at_unpack.argtypes = [vp, d, ll, vp, vp, ll, vp, i32, vp, i32]
        L.emul_endpoint_position.argtypes = [ll, i32, i32, i32, i32, i32, i32]
        L.emul_endpoint_position.restype = ll
        for f in (L.emul_at_update, L.emul_at_arm, L.emul_at_clear, L.emul_at_arm_at, L.emul_at_pack, L.emul_at_unpack):
            f.restype = None
        _emul.append(L)
    return _emul[0]


class Emul(TE.Emul):
    """TE.Emul (the C-ABI's host logic over the plain bodies) plus the positioned mode: the mute words, the reduction keys and
    the switch to the positioned bodies at the first arm_at"""

    def __init__(self, *args, order_seed=None, **kw):
        super().__init__(*args, **kw)
        n = self.members.size
        self.mute = np.zeros(max(n, 1), np.int32)
        self.key = np.zeros(max(n, 1), np.uint64)
        self.positioned = False
        self.rng = np.random.default_rng(order_seed) if order_seed is not None else None
        self.launches = 0

    def _cm(self):
        return self._c() + (self.mute.ctypes.data,)

    def update(self, probs, S, buffered, pending):
        if not self.positioned:
            return super().update(probs, S, buffered, pending)
        probs = np.ascontiguousarray(probs, np.float32)
        n = probs.shape[1]
        if not emul().emul_endpoint_fits(self.base[0], self.base[1], self.base[2], S, buffered, pending, self.hop, self.stride, n):
            raise ValueError("inconsistent update")
        pos0 = emul().emul_endpoint_position(S, buffered, self.hop, pending, self.stride, n, 0)
        emul().emul_at_update(*self._cm(), probs.ctypes.data, n, n, pos0)
        self.base = (S, buffered, pending)
        keep = min(n, 64)
        self.pos[keep:] = self.pos[:64 - keep].copy()
        self.pos[:keep] = pos0 + (n - 1 - np.arange(keep)) * self.step_samples
        self.steps += n

    def arm(self, ids):
        if not self.positioned:
            return super().arm(ids)
        ids = np.ascontiguousarray(ids, np.int32)
        self.tag += 1
        emul().emul_at_arm(*self._cm(), ids.ctypes.data, ids.size, min(self.lookback, self.steps), self.tag, self.pos.ctypes.data)

    def clear(self, ids, reset, counters=None):
        if not self.positioned:
            return super().clear(ids, reset, counters)
        if ids is None:
            emul().emul_at_clear(*self._cm(), None, self.members.size, reset)
            self.base, self.steps, self.pos = tuple(counters), 0, np.zeros(64, np.int64)
        else:
            ids = np.ascontiguousarray(ids, np.int32)
            emul().emul_at_clear(*self._cm(), ids.ctypes.data, ids.size, reset)

    def disarm(self, ids):
        self.clear(ids, 0)

    def reset(self, ids=None, counters=None):
        self.clear(ids, 1, counters)

    def q(self):
        S, b, g = self.base
        return emul().emul_endpoint_position(S, b, self.hop, g, self.stride, 1, 0)

    def arm_at(self, ids, positions, skip):
        self.positioned = True
        ids = np.ascontiguousarray(ids, np.int32)
        P = np.ascontiguousarray(positions, np.int64)
        order = np.ascontiguousarray(self.rng.permutation(ids.size) if self.rng is not None else np.arange(ids.size), np.int32)
        self.tag += 1
        emul().emul_at_arm_at(*self._cm(), self.key.ctypes.data, ids.ctypes.data, P.ctypes.data, ids.size, order.ctypes.data,
                              min(self.lookback, self.steps), self.tag, self.pos.ctypes.data, self.q(), skip)
        assert not self.key.any()                                  # every key is back to "none" for the next call

    def state(self):
        st = super().state()
        st["mute"] = self.mute[:self.members.size].copy()
        return st


def same(a, b):
    return TE.same_state(a, b) and np.array_equal(np.asarray(a["mute"]), np.asarray(b["mute"]))


def pair(n_streams, members, counters, **rule):
    return [A.EndpointAtRef(n_streams, members, 3, 160, counters=counters, **rule), Emul(n_streams, members, 3, 160, counters=counters, **rule)]


def live(objs, fe, probs):
    """one 480-sample live call per column of probs"""
    for j in range(probs.shape[1]):
        fe.call(480)
        for o in objs:
            o.update(probs[:, j:j + 1], *fe.counters())


def check(objs):
    ref, em = objs
    assert same(ref.state(), em.state()), (ref.state(), em.state())
    (er, nr), (ee, ne) = ref.drain(), em.drain()
    assert nr == ne and np.array_equal(TE.sort_events(er), TE.sort_events(ee)), (er, ee)
    return TE.sort_events(er)


RULE1 = dict(TE.RULE, vad_window=1, lookback_steps=20)


def one_row(flags, ops, **kw):
    """one stream of 0 / 1 flags (window 1) in live calls, with ops {step: [(name, args)]} before that step's call"""
    rule = dict(RULE1, **kw)
    fe = TE.Frontend(buffered=320)                       # step j of the live calls ends at 480 (j + 1)
    objs = pair(1, [0], fe.counters(), **rule)
    for j, f in enumerate(list(flags) + [None]):
        for name, args in ops.get(j, []):
            for o in objs:
                getattr(o, name)(*args)
        if f is None:
            break
        live(objs, fe, np.array([[1.0 if f else 0.0]], np.float32))
    return objs


# ---- positions and skips -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [480 * 8, 480 * 8 + 1, 480 * 8 - 1, 480 * 3 + 200, 480 * 12, 480 * 12 + 5000, 480 * 2, -7000])
@pytest.mark.parametrize("skip", [0, 480, 960 * 3 + 17])
def test_one_row_positions_and_skips_match_the_rule(P, skip):
    """P on and between grid points, at the newest step, in the future, older than the replay (lookback 4) and negative"""
    rng = np.random.default_rng(P % 1000 + skip)
    flags = (rng.random(40) < 0.6).tolist()
    for lookback in (4, 20):
        objs = one_row(flags, {12: [("arm_at", ([0], [P], skip))]}, lookback_steps=lookback, silence_steps=4, timeout_steps=30, max_steps=60)
        check(objs)


def test_mute_spans_several_updates_and_the_stored_flags_keep_the_truth():
    skip = 480 * 5 + 100                                  # 5 future steps muted
    objs = one_row([1] * 30, {10: [("arm_at", ([0], [480 * 10], skip))]}, silence_steps=3, timeout_steps=100)
    st = objs[1].state()
    assert int(st["flags"][0]) == (1 << 30) - 1           # every stored flag 1
    assert int(st["elapsed"][0]) == 20 and int(st["heard"][0]) == 1
    assert int(st["start_sample"][0]) == 480 * 10
    check(objs)
    # a mute that is still running: look at it after two of its steps
    objs = one_row([1] * 12, {10: [("arm_at", ([0], [480 * 10], skip))]})
    assert objs[1].state()["mute"][0] == objs[0].state()["mute"][0] == 3
    check(objs)


def test_run_on_speech_inside_the_skip_is_not_the_command():
    """the wake word's tail runs past P: inside the skip it does not count, so a pause after it cannot end the command"""
    flags = [0] * 5 + [1] * 10 + [0] * 12 + [1] * 20 + [0] * 10     # wake word, pause of 12 steps, command, silence
    P = 480 * 13                                                  # detection two steps before the wake word's speech ends
    plain = one_row(flags, {40: [("arm", ([0],))]}, lookback_steps=40, silence_steps=8, timeout_steps=100)
    (ev, _), _ = plain[0].drain(), plain[1].drain()
    assert ev["reason"].tolist() == [R.END_OF_SPEECH] and ev["speech_end_sample"][0] == 480 * 15      # ended after the wake word
    at = one_row(flags, {40: [("arm_at", ([0], [P], 480 * 3))]}, lookback_steps=40, silence_steps=8, timeout_steps=100)
    ev = check(at)
    assert ev["reason"].tolist() == [R.END_OF_SPEECH]
    assert ev["start_sample"][0] == P and ev["speech_end_sample"][0] == 480 * 47                     # ended after the command


def test_an_end_reached_during_the_replay_is_emitted_by_the_arm():
    objs = one_row([0] * 30, {30: [("arm_at", ([0], [480 * 5], 0))]}, lookback_steps=30, timeout_steps=10)
    ev = check(objs)
    assert ev["reason"].tolist() == [R.NO_SPEECH] and ev["end_sample"][0] == 480 * 15 and ev["start_sample"][0] == 480 * 5
    assert objs[1].state()["mute"][0] == 0 and objs[1].state()["armed"][0] == -1


@pytest.mark.parametrize("op", ["arm", "disarm", "reset"])
def test_arm_disarm_and_reset_mid_mute_clear_it(op):
    args = ([0],)
    objs = one_row([1, 0] * 15, {10: [("arm_at", ([0], [480 * 10], 480 * 8))], 13: [(op, args)]}, timeout_steps=100)
    assert objs[1].state()["mute"][0] == 0
    check(objs)


def test_duplicate_ids_arm_once_at_the_latest_position_in_any_order():
    rng = np.random.default_rng(3)
    members = [1, 2, 4, 6]
    for trial in range(8):
        fe = TE.Frontend(buffered=320)
        objs = [A.EndpointAtRef(8, members, 3, 160, counters=fe.counters(), **dict(TE.RULE, lookback_steps=30)),
                Emul(8, members, 3, 160, counters=fe.counters(), order_seed=trial, **dict(TE.RULE, lookback_steps=30))]
        live(objs, fe, TE._tracks(rng, 4, 25))
        ids = rng.choice([1, 2, 4, 6, 0, 3, -1, 9], 12)
        pos = rng.choice([480 * 10, 480 * 15, 480 * 15 + 7, 480 * 30, 480 * 20], 12)
        skip = int(rng.choice([0, 480, 2000]))
        for o in objs:
            o.arm_at(ids, pos, skip)
        live(objs, fe, TE._tracks(rng, 4, 15))
        check(objs)


def test_no_steps_after_a_whole_reset():
    """q is where the newest step would have been; the start stays at P' through the first update (the placed bit)"""
    objs = one_row([1] * 6, {})
    for o in objs:
        o.reset(None, (0, 320, 0))
        o.arm_at([0], [-100], 0)
    assert objs[1].state()["mute"][0] == A.PLACED == objs[0].state()["mute"][0]
    for o in objs:
        o.update(np.array([[0.0]], np.float32), 480, 320, 0)
    st = objs[1].state()
    assert int(st["start_sample"][0]) == -100 and int(st["elapsed"][0]) == 1 and st["mute"][0] == 0
    check(objs)
    objs = one_row([1] * 6, {})
    for o in objs:
        o.reset(None, (0, 320, 0))
        o.arm_at([0], [5000], 800)                      # in the future: P' = q = 0, and one step muted
    assert objs[1].state()["mute"][0] == A.PLACED + 1
    for o in objs:
        o.update(np.array([[1.0]], np.float32), 480, 320, 0)
    assert int(objs[1].state()["start_sample"][0]) == 0 and int(objs[1].state()["run"][0]) == 0
    check(objs)


# ---- the properties ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_property_1_arm_at_one_step_before_the_replay_is_arm(seed):
    rng = np.random.default_rng(seed)
    lookback = int(rng.choice([1, 5, 10, 64]))
    fe = TE.Frontend(buffered=320)
    plain = Emul(6, [0, 2, 3, 5], 3, 160, counters=fe.counters(), **dict(TE.RULE, lookback_steps=lookback))
    at = Emul(6, [0, 2, 3, 5], 3, 160, counters=fe.counters(), **dict(TE.RULE, lookback_steps=lookback))
    at.positioned = True
    probs = TE._tracks(rng, 4, 120)
    for j in range(120):
        fe.call(480)
        for o in (plain, at):
            o.update(probs[:, j:j + 1], *fe.counters())
        if j % 17 == 16:
            L = min(lookback, plain.steps)
            P = int(plain.pos[L - 1]) - plain.step_samples
            plain.arm([0, 2, 5])
            at.arm_at([0, 2, 5], [P] * 3, 0)
            assert same(plain.state(), at.state()) and (at.state()["mute"] == 0).all()
    (ea, na), (eb, nb) = plain.drain(), at.drain()
    assert na == nb > 0 and np.array_equal(TE.sort_events(ea), TE.sort_events(eb))


@pytest.mark.parametrize("seed", range(4))
def test_property_2_results_do_not_depend_on_when_arm_at_is_called(seed):
    rng = np.random.default_rng(100 + seed)
    probs = TE._tracks(rng, 3, 90)
    skip = int(rng.choice([0, 480 * 4 + 3, 480 * 9]))
    P = 480 * 30 + int(rng.integers(-400, 400))
    outs = []
    for late in (31, 34, 40, 45):                        # the replay of 20 steps still reaches P at step 45
        objs = [A.EndpointAtRef(3, [0, 1, 2], 3, 160, counters=(0, 320, 0), **dict(TE.RULE, lookback_steps=20)),
                Emul(3, [0, 1, 2], 3, 160, counters=(0, 320, 0), **dict(TE.RULE, lookback_steps=20))]
        fe = TE.Frontend(buffered=320)
        live(objs, fe, probs[:, :late])
        for o in objs:
            o.arm_at([0, 1, 2], [P] * 3, skip)
        live(objs, fe, probs[:, late:])
        outs.append(objs[0].state())
        ev = check(objs)
        outs[-1]["events"] = ev
    for o in outs[1:]:
        assert same(o, outs[0]) and np.array_equal(o["events"], outs[0]["events"])


@pytest.mark.parametrize("seed", range(4))
def test_property_3_positioned_forms_with_zero_mutes_are_the_plain_forms(seed):
    """the random tracks of test_endpoint, split into calls anywhere, through the plain bodies and the positioned ones"""
    rng = np.random.default_rng(seed)
    n_streams, total = 24, 250
    members = np.sort(rng.choice(n_streams, 17, replace=False)).astype(np.int32)
    probs = TE._tracks(rng, members.size, total)
    ops = {}
    for at in sorted(rng.choice(np.arange(1, total), 30, replace=False).tolist()):
        kind = str(rng.choice(["arm", "arm", "disarm", "reset", "drain"]))
        ops.setdefault(int(at), []).append((kind, rng.integers(-2, n_streams + 2, 6).astype(np.int32) if kind == "arm"
                                            else rng.integers(0, n_streams, 2).astype(np.int32)))
    ops.setdefault(0, []).append(("arm", members))
    runs = []
    for positioned in (False, True):
        fe = TE.Frontend(160, 3, seen=1000)
        em = Emul(n_streams, members, 3, 160, counters=fe.counters(), **dict(TE.RULE, lookback_steps=10))
        em.positioned = positioned
        drains = TE._drive_exact(em, fe, probs, ops, TE.SPLITS["mixed"], np.random.default_rng(seed))
        runs.append(([TE.sort_events(x[0]) for x in drains], em.state()))
    assert all(np.array_equal(a, b) for a, b in zip(runs[0][0], runs[1][0])) and same(runs[0][1], runs[1][1])


@pytest.mark.parametrize("seed", range(4))
def test_random_positioned_sessions_match_the_rule_however_split(seed):
    """arm_at beside arm, disarm and reset, positions spread around the replay, through two splits into calls"""
    rng = np.random.default_rng(50 + seed)
    n_streams, total = 16, 260
    members = np.sort(rng.choice(n_streams, 11, replace=False)).astype(np.int32)
    probs = TE._tracks(rng, members.size, total)
    script = {}
    for at in sorted(rng.choice(np.arange(5, total), 35, replace=False).tolist()):
        kind = str(rng.choice(["arm_at", "arm_at", "arm_at", "arm", "disarm", "reset", "drain"]))
        ids = rng.integers(-2, n_streams + 2, 5).astype(np.int32)
        script[int(at)] = (kind, ids, rng.integers(-3000, 4000, 5), int(rng.choice([0, 480, 2400, 7000])))
    results = []
    for splits in ("live", "mixed"):
        for cls in (A.EndpointAtRef, Emul):
            fe = TE.Frontend(160, 3, seen=5000)
            obj = cls(n_streams, members, 3, 160, counters=fe.counters(), **dict(TE.RULE, lookback_steps=12))
            srng = np.random.default_rng(seed)
            used, drains = 0, []
            for stop in sorted(script) + [total]:
                while used < stop:
                    n16 = int(srng.choice(TE.SPLITS[splits]))
                    if used + TE._steps_of(fe, n16) > stop:
                        n16 = fe.hop
                    steps, _ = fe.call(n16)
                    obj.update(probs[:, used:used + steps], *fe.counters())
                    used += steps
                if stop == total:
                    break
                kind, ids, offs, skip = script[stop]
                q = obj.q()
                if kind == "arm_at":
                    obj.arm_at(ids, q + offs * 3, skip)
                elif kind == "drain":
                    drains.append(TE.sort_events(obj.drain()[0]))
                elif kind == "arm":
                    obj.arm(ids)
                else:
                    ok = ids[(ids >= 0) & (ids < n_streams)]
                    getattr(obj, kind)(ok)
            drains.append(TE.sort_events(obj.drain()[0]))
            results.append((drains, obj.state()))
    base = results[0]
    assert sum(x.size for x in base[0]) > 5
    for drains, st in results[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(drains, base[0]))
        assert same(dict(st, samples_seen=base[1]["samples_seen"], buffered=base[1]["buffered"], pending=base[1]["pending"]), base[1])


# ---- records -----------------------------------------------------------------------------------------------------------------------
def test_records_carry_the_mute_word_and_plain_records_stay_plain():
    rng = np.random.default_rng(9)
    members = [0, 1, 2, 3]
    fe = TE.Frontend(buffered=320)
    em = Emul(5, members, 3, 160, counters=fe.counters(), **dict(TE.RULE, lookback_steps=20))
    live([em], fe, TE._tracks(rng, 4, 30))
    em.arm([0])
    plain_before = np.zeros((5, emul().emul_at_record_bytes(5) // 4), np.uint32)
    ids = np.arange(5, dtype=np.int32)
    emul().emul_at_pack(*em._cm(), em.base[0], ids.ctypes.data, 5, plain_before.ctypes.data, 0)
    positioned_zero = np.zeros_like(plain_before)
    emul().emul_at_pack(*em._cm(), em.base[0], ids.ctypes.data, 5, positioned_zero.ctypes.data, 1)
    assert np.array_equal(plain_before, positioned_zero)                  # with every mute 0 the records are the plain ones
    em.arm_at([1, 2], [em.q() - 480 * 2, em.q()], 480 * 7)
    rec = np.zeros_like(plain_before)
    emul().emul_at_pack(*em._cm(), em.base[0], ids.ctypes.data, 5, rec.ctypes.data, 1)
    assert rec[1, 2] == em.mute[1] == 5 and rec[2, 2] == em.mute[2] == A.PLACED + 7 and rec[0, 2] == 0 and rec[4].sum() == 0
    # into a positioned endpointer on a younger axis: the words land with the rows, rebased
    dst = Emul(5, members, 3, 160, counters=(0, 320, 0), **dict(TE.RULE, lookback_steps=20))
    dst.positioned = True
    dst.mute[:] = 99
    emul().emul_at_unpack(*dst._cm(), 0, ids.ctypes.data, 5, rec.ctypes.data, 1)
    assert dst.mute.tolist() == [0, 5, A.PLACED + 7, 0]
    assert int(dst.a["start"][2]) == em.q() - em.base[0]
    # plain records into a positioned endpointer: mute 0
    dst.mute[:] = 99
    emul().emul_at_unpack(*dst._cm(), 0, ids.ctypes.data, 5, plain_before.ctypes.data, 1)
    assert (dst.mute == 0).all()


# ---- build, ABI and refusals ----------------------------------------------------------------------------------------------------------
NEW = {"mww_endpointer_arm_at": ("mww_endpointer_t *ep, const int32_t *h_ids, const int64_t *h_positions, int n, long long skip_samples, "
                                 "void *cu_stream", [vp, vp, vp, i32, ll, vp]),
       "mww_endpointer_arm_at_device": ("mww_endpointer_t *ep, const int32_t *d_ids, const int64_t *d_positions, int n, long long skip_samples, "
                                        "void *cu_stream", [vp, vp, vp, i32, ll, vp]),
       "mww_endpointer_get_mutes": ("mww_endpointer_t *ep, int32_t *h_mutes", [vp, vp]),
       "mww_endpointer_set_mutes": ("mww_endpointer_t *ep, const int32_t *h_mutes", [vp, vp])}


def test_new_symbols_are_declared_and_exported_with_their_arguments():
    from microwakeword_b200 import _lib, build
    L = _lib.lib()
    syms = subprocess.run(["nm", "-D", "--defined-only", build.OUT], capture_output=True, text=True, check=True).stdout
    hdr = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "mww.h")).read())
    for name, (sig, args) in NEW.items():
        assert name in _lib.EXPORTS and re.search(r"\bT %s\b" % name, syms), name
        assert "int %s(%s);" % (name, sig) in hdr, name
        assert getattr(L, name).argtypes == args, name
    assert ctypes.sizeof(_lib.MwwEndpointerLayout) == 48 and ctypes.sizeof(_lib.MwwEndpointState) == 10 * 8 + 4 * 8 + 64 * 8


def test_null_endpointers_are_refused_without_device_work():
    from microwakeword_b200 import _lib
    L = _lib.lib()
    assert L.mww_endpointer_arm_at(None, None, None, 0, 0, None) == -1 and b"NULL" in L.mww_last_error(None)
    assert L.mww_endpointer_arm_at_device(None, None, None, 0, 0, None) == -1
    assert L.mww_endpointer_get_mutes(None, None) == -1 and L.mww_endpointer_set_mutes(None, None) == -1


def test_python_refusals_before_the_library_is_called():
    from microwakeword_b200.endpoint import Endpointer

    class Eng:
        _h, device, n_streams, audio_history_capacity = ctypes.c_void_p(1), 0, 8, 1600

    class Det:                                            # the parts of a detector arm(at=) reads
        def __init__(self, timed=True, device=0, engine=None):
            self.timed, self.device, self.capacity, self.engine = timed, device, 4, engine
            self.fired_ids = self.event_samples = object()

    ep = object.__new__(Endpointer)
    ep.__dict__.update(_L=TE.NoLib(), device=0, capacity=8, n_rows=4, engine=Eng(), vad_window=5, stride=3, hop=160)
    cases = [
        (dict(ids=[0], at=None, skip=0), "skip applies"),
        (dict(ids=[0], at=[0], skip=-1), "skip"),
        (dict(ids=[0], at=[0], skip=(1 << 22) + 1), "skip"),
        (dict(ids=[0], at=[0], skip=1.5), "integer"),
        (dict(ids=[0], at=Det(timed=False)), "timed"),
        (dict(ids=[0], at=Det(device=1)), "cuda:1"),
        (dict(ids=[0], at=Det(engine=Eng())), "another engine"),
        (dict(ids=[0], at=Det()), "CUDA int32 tensor of its 4 slots"),
        (dict(ids=[0, 1], at=[0]), "beside the ids"),
        (dict(ids=[0], at=[0.5]), "integer sequence"),
        (dict(ids=[8], at=[0]), "stream ids"),
        (dict(ids=[0], at=np.zeros((1, 1), np.int64)), "1-D"),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            ep.arm(**kw)


def _cuobjdump():
    from microwakeword_b200 import _lib, build
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed next to nvcc")
    _lib.lib()
    return tool


def test_every_existing_kernel_keeps_its_instructions():
    from microwakeword_b200 import build
    from test_event_positions import _sass_hashes
    before = json.load(open(os.path.join(GOLDEN, "sass_kernels_before_endpoint_at.json")))
    libs = [k for k in before if k != "_comment"]
    assert len(libs) == 19 and "libmww_endpoint.so" in libs and "libmww_serving_records.so" in libs
    _cuobjdump()
    for lib in libs:
        assert _sass_hashes(os.path.join(os.path.dirname(build.OUT), lib)) == before[lib], lib


def test_companion_library_holds_exactly_its_kernels_without_stack_local_memory_or_spills(monkeypatch):
    from microwakeword_b200 import build
    assert os.path.basename(build.EPA_OUT) == "libmww_endpoint_at.so" and build.EPA_SOURCES == ["mww_endpoint_at.cu"]
    res = subprocess.run([_cuobjdump(), "-res-usage", build.EPA_OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res)
    names = [n for n, *_ in found]
    assert len(names) == 7, res
    for k in ("endpoint_update_muted_kernel", "endpoint_arm_muted_kernel", "endpoint_clear_muted_kernel", "endpoint_at_reduce_kernel",
              "endpoint_arm_at_kernel", "pack_endpointer_rows_muted_kernel", "unpack_endpointer_rows_muted_kernel"):
        assert sum(re.search(r"\d%s" % k, n) is not None for n in names) == 1, k
    assert all(int(stack) == int(local) == int(shared) == 0 for _, _, stack, shared, local in found), found
    flags = [f for f in build.FLAGS if f not in ("-shared", "-cudart", "static")]
    rep = subprocess.run([build.NVCC] + flags + ["-cubin", "-Xptxas", "-v", "-o", os.path.join(_BUILD.name, "at.cubin"),
                                                 os.path.join(CSRC, "mww_endpoint_at.cu")], capture_output=True, text=True, check=True).stderr
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rep)
    assert len(spills) == 7 and all(int(a) == int(b) == int(c) == 0 for a, b, c in spills), rep
    dyn = subprocess.run(["readelf", "-d", build.OUT], capture_output=True, text=True).stdout
    assert "[libmww_endpoint_at.so]" in dyn
    real = os.path.exists
    monkeypatch.setattr(build.os.path, "exists", lambda p: p != build.EPA_OUT and real(p))
    assert build._stale()


def test_timing_tool_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    tool = os.path.join(ROOT, "tools", "endpoint_at_time.py")
    res = subprocess.run([sys.executable, tool, "--rounds", "1"], capture_output=True, text=True)
    assert res.returncode != 0 and "CUDA" in res.stderr
