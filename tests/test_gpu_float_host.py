"""float32 HOST audio through the staged pipeline (run with -m gpu on an H100).

mww_predict_clip_host[_multi]_f32 and mww_predict_clip_remote[_multi]_f32 (StreamEngine / MultiModelEngine predict_clip_host
with a float32 array, predict_clip_remote with dtype=float32, Model.step with float32 numpy) copy the float samples as they are
and convert them in the frontend kernels.  Their contract is that of the device float entry points: exactly what the int16
call gives on audio_utils.to_int16 of the same audio -- bit-identical probabilities and state_dict() after every call -- for
fp32, int8 and run-time-geometry models, one-model and multi-model handles, with int16 and float32 calls alternating on one
handle.  Every float call here runs on one handle and the int16 call on to_int16 of the same samples on a twin handle.

Audio: P distinct base streams of random float audio (per-stream amplitudes from -80 dBFS to clipping), salted with every
float within 2 ulp of an integer boundary, NaNs, infinities, subnormals, +-0 and +-FLT_MAX; stream s carries base[s % P]."""

import ast
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from microwakeword_b200 import _lib
from microwakeword_b200.audio.audio_utils import to_int16

pytestmark = pytest.mark.gpu

P = 1021                       # prime: neighbouring tiles and CTAs see different audio
N_TOTAL = 48000 + 48000 + 47999 + 48001
BIG = 65536


def _salt(rng):
    k = rng.integers(-32770, 32771, 4096)
    centre = (k / 32768.0).astype(np.float32)
    near = [centre]
    for direction in (np.inf, -np.inf):
        x = centre
        for _ in range(2):
            x = np.nextafter(x, np.float32(direction))
            near.append(x)
    special = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, np.finfo(np.float32).max, -np.finfo(np.float32).max,
                                        0.99999994, 3.0517578e-05], np.float32),
                              np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FA5A5A5, 0x00000001, 0x807FFFFF],
                                       np.uint32).view(np.float32)])
    return np.concatenate(near + [np.repeat(special, 64)])


def make_audio():
    """(base float32 [P, N_TOTAL], its to_int16 [P, N_TOTAL]), host arrays"""
    rng = np.random.default_rng(43)
    amp = (10.0 ** rng.uniform(-4.0, 0.3, P)).astype(np.float32)[:, None]       # -80 dBFS .. 2x full scale (clipping)
    base = (rng.standard_normal((P, N_TOTAL), dtype=np.float32) * amp).astype(np.float32)
    salt = _salt(rng)
    pos = rng.random((P, N_TOTAL)) < 0.02
    base[pos] = salt[rng.integers(0, salt.size, int(pos.sum()))]
    with np.errstate(invalid="ignore", over="ignore"):
        i16 = to_int16(base)
    return base, i16


@pytest.fixture(scope="module")
def audio():
    return make_audio()


def fill(dst, base, pos):
    """dst [S, n] (any host buffer, any row pitch) <- stream s carries base[s % P, pos:pos + n]; returns dst"""
    S, n = dst.shape
    for s0 in range(0, S, P):
        k = min(P, S - s0)
        dst[s0:s0 + k] = base[:k, pos:pos + n]
    return dst


def chunk(base, S, pos, n):
    return fill(np.empty((S, n), base.dtype), base, pos)


def blob(name):
    with open(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % name), "rb") as f:
        return f.read()


def as_np(r):
    return r.cpu().numpy() if hasattr(r, "cpu") else np.asarray(r)


def same_state(a, b, where=""):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            same_state(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(a, list):
        assert len(a) == len(b), where
        for k, (x, y) in enumerate(zip(a, b)):
            same_state(x, y, "%s[%d]" % (where, k))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), where
    else:
        assert a == b, where


def same_probs(got, want, what):
    got, want = (got, want) if isinstance(got, list) else ([got], [want])
    assert len(got) == len(want), what
    for k, (g, w) in enumerate(zip(got, want)):
        g, w = as_np(g), as_np(w)
        assert g.dtype == w.dtype == np.float32 and g.shape == w.shape, (what, k, g.shape, w.shape)
        assert np.array_equal(g.view(np.int32), w.view(np.int32)), (what, k)


class Twin:
    """`f` takes the float32 calls (and the int16 calls of an alternating schedule), `i` the int16 calls on to_int16 of the
    same samples; after every call the probabilities and both handles' state_dict() must be bit-identical"""

    def __init__(self, make):
        self.f, self.i = make(), make()

    def check(self, on_f, on_i, what):
        same_probs(on_f(self.f), on_i(self.i), what)
        same_state(self.f.state_dict(), self.i.state_dict(), what)


def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- 65 536 streams: the benchmark's shape --------------------------------------------------------------------------------

@pytest.mark.parametrize("model", ["f32", "int8"])
def test_host_clip_calls_at_65536_streams(torch_cuda, audio, model):
    """two 3 s calls (the second enters with 320 carried samples), then 47 999 and 48 001 samples"""
    from microwakeword_b200.engine import StreamEngine
    base_f, base_i = audio
    t = Twin(lambda: StreamEngine(blob(model), n_streams=BIG))
    flat_f, flat_i = np.empty(BIG * 48001, np.float32), np.empty(BIG * 48001, np.int16)     # 12.6 + 6.3 GB, reused
    pos = 0
    for n in (48000, 48000, 47999, 48001):
        x_f = fill(flat_f[:BIG * n].reshape(BIG, n), base_f, pos)
        x_i = fill(flat_i[:BIG * n].reshape(BIG, n), base_i, pos)
        t.check(lambda e: e.predict_clip_host(x_f), lambda e: e.predict_clip_host(x_i), ("host", model, n))
        pos += n
    assert pos == N_TOTAL


# ---- buffer kinds and row pitches --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("model", ["f32", "int8"])
def test_row_pitch_pinned_and_write_combined_buffers(torch_cuda, audio, model):
    """float32 from a column slice of a wider pageable array (row pitch != n: the 2-D copy), a pinned array and a column slice
    of one, and a write-combined input buffer; clip and live calls in turn on one handle"""
    from microwakeword_b200.engine import StreamEngine, host_array
    base_f, base_i = audio
    S = 6 * sms(torch_cuda) + 37
    t = Twin(lambda: StreamEngine(blob(model), n_streams=S))
    kinds = {
        "pageable": lambda n: np.empty((S, n), np.float32),
        "pageable_slice": lambda n: np.empty((S, n + 13), np.float32)[:, 5:5 + n],
        "pinned": lambda n: host_array((S, n), np.float32),
        "pinned_slice": lambda n: host_array((S, n + 8), np.float32)[:, 3:3 + n],
        "write_combined": lambda n: host_array((S, n), np.float32, write_combined=True),
    }
    pos = 0
    for kind, make in kinds.items():
        for n in (16001, 480, 480):
            x_f = fill(make(n), base_f, pos)
            if kind.endswith("slice"):
                assert not x_f.flags.c_contiguous and x_f.strides[1] == 4
            x_i = chunk(base_i, S, pos, n)
            t.check(lambda e: e.predict_clip_host(x_f), lambda e: e.predict_clip_host(x_i), (kind, n))
            pos += n
    assert pos <= N_TOTAL


# ---- many tiles: MWW_SCRATCH_MB is read at create, so this runs in a child process ---------------------------------------

SCRATCH_MB = 8


def child_many_tiles():
    """-> 'OK <tiles per call>' or 'FAIL <why>'.  Run with MWW_SCRATCH_MB=SCRATCH_MB set before the handles are created."""
    import torch
    from microwakeword_b200.engine import StreamEngine
    base_f, base_i = make_audio()
    S = 6 * sms(torch) + 37
    budget = SCRATCH_MB << 20
    tiles = []
    try:
        for model in ("f32", "int8"):
            t = Twin(lambda: StreamEngine(blob(model), n_streams=S))
            t.f.profile(True)
            pos = 0
            for n in (48000, 47999, 480):
                x_f, x_i = chunk(base_f, S, pos, n), chunk(base_i, S, pos, n)
                frames = (t.f.frontend_buffered + n - 480) // 160 + 1
                launches = t.f.launch_count
                t.check(lambda e: e.predict_clip_host(x_f), lambda e: e.predict_clip_host(x_i), (model, n))
                got = t.f.timeline_read().shape[0]          # tiles of the last staged call
                # the two float32 staging tiles count against the budget with the feature scratch (and the K1 -> K2
                # scratch when the clip kernel is not fused)
                want = {-(-S // max(1, budget // (2 * 4 * n + frames * 40 * scratch))) for scratch in (2, 6)}
                if got not in want:
                    return "FAIL %s %d samples: %d tiles, expected one of %s" % (model, n, got, sorted(want))
                if t.f.launch_count - launches < 2 * got:       # at least the frontend and the model in every tile
                    return "FAIL %s %d samples: %d launches for %d tiles" % (model, n, t.f.launch_count - launches, got)
                tiles.append(got)
                pos += n
    except AssertionError as e:
        return "FAIL %r" % (e.args,)
    return "OK %s" % tiles


def test_many_tiles_from_the_scratch_budget():
    env = dict(os.environ, MWW_SCRATCH_MB=str(SCRATCH_MB))
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_float_host as T; print('VERDICT', T.child_many_tiles())"
            % (ROOT, os.path.join(ROOT, "tests")))
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable] + flags + ["-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("VERDICT ")]
    assert res.returncode == 0 and len(lines) == 1, (res.returncode, res.stdout[-2000:], res.stderr[-4000:])
    verdict = lines[0][len("VERDICT "):]
    assert verdict.startswith("OK "), verdict
    assert max(ast.literal_eval(verdict[3:])) > 16, verdict       # more tiles than the default pipeline's 16


# ---- predict_clip_remote with dtype=float32 ----------------------------------------------------------------------------------

def test_remote_float32_from_host_and_from_this_gpu(torch_cuda, audio):
    """host source at tiles=0 (staged, 16 tiles) and tiles=16; this GPU's own memory at tiles=16 (staged) and tiles=0 (read in
    place by the device float path)"""
    from microwakeword_b200.engine import StreamEngine, host_array
    torch = torch_cuda
    base_f, base_i = audio
    S = 6 * sms(torch) + 37
    for model in ("f32", "int8"):
        t = Twin(lambda: StreamEngine(blob(model), n_streams=S))
        pos = 0
        for source, tiles, n in (("host", 0, 48000), ("host", 16, 47999), ("device", 16, 48001), ("device", 0, 480), ("host", 16, 480)):
            if source == "host":
                x_f, x_i = fill(host_array((S, n), np.float32), base_f, pos), fill(host_array((S, n), np.int16), base_i, pos)
                p_f, p_i = x_f.ctypes.data, x_i.ctypes.data
            else:
                x_f, x_i = torch.from_numpy(chunk(base_f, S, pos, n)).cuda(), torch.from_numpy(chunk(base_i, S, pos, n)).cuda()
                p_f, p_i = x_f.data_ptr(), x_i.data_ptr()
            t.check(lambda e: e.predict_clip_remote(p_f, n, tiles=tiles, dtype=np.float32),
                    lambda e: e.predict_clip_remote(p_i, n, tiles=tiles), (model, source, tiles, n))
            torch.cuda.synchronize()                                 # the sources stay alive until the calls are done
            pos += n


# ---- several models over one frontend --------------------------------------------------------------------------------------

def test_multi_model_host_and_remote_float32(torch_cuda, audio):
    """fp32 and int8 okay_nabu and a run-time geometry of stride 17 on one frontend; every model against its int16 counterpart"""
    from generic_range import GEOMETRIES, models as range_models
    from microwakeword_b200 import model_file as MF
    from microwakeword_b200.engine import MultiModelEngine, host_array
    torch = torch_cuda
    base_f, base_i = audio
    S = 6 * sms(torch) + 37
    blobs = [blob("f32"), blob("int8"), MF.write_container(range_models(GEOMETRIES["long_stride"])[0])]
    t = Twin(lambda: MultiModelEngine(blobs, n_streams=S))
    pos = 0
    for how, n in (("host", 48000), ("host_slice", 47999), ("remote_host", 48001), ("remote_device", 16000), ("host", 480),
                   ("remote_host", 480)):
        x_i = chunk(base_i, S, pos, n)
        if how == "host_slice":
            x_f = fill(np.empty((S, n + 3), np.float32)[:, 1:1 + n], base_f, pos)
        elif how == "remote_host":
            x_f = fill(host_array((S, n), np.float32), base_f, pos)
        else:
            x_f = chunk(base_f, S, pos, n)
        if how.startswith("host"):
            t.check(lambda e: e.predict_clip_host(x_f), lambda e: e.predict_clip_host(x_i), (how, n))
        elif how == "remote_host":
            t.check(lambda e: e.predict_clip_remote(x_f.ctypes.data, n, dtype=np.float32), lambda e: e.predict_clip_host(x_i), (how, n))
        else:
            d_f = torch.from_numpy(x_f).cuda()
            t.check(lambda e: e.predict_clip_remote(d_f.data_ptr(), n, tiles=5, dtype=torch.float32), lambda e: e.predict_clip_host(x_i),
                    (how, n))
        torch.cuda.synchronize()
        pos += n


# ---- live steps, int16 and float32 alternating ---------------------------------------------------------------------------

@pytest.mark.parametrize("model", ["f32", "int8"])
def test_live_host_steps_alternating_int16_and_float32(torch_cuda, audio, model):
    from microwakeword_b200.engine import StreamEngine
    base_f, base_i = audio
    S = 6 * sms(torch_cuda) + 37
    t = Twin(lambda: StreamEngine(blob(model), n_streams=S))
    pos = 0
    for step in range(56):
        x_i = chunk(base_i, S, pos, 480)
        x_f = chunk(base_f, S, pos, 480) if step % 2 == 0 else x_i
        same_probs(t.f.predict_clip_host(x_f), t.i.predict_clip_host(x_i), (model, step))
        if step % 8 == 7:
            same_state(t.f.state_dict(), t.i.state_dict(), (model, step))
        pos += 480


# ---- Model.step ---------------------------------------------------------------------------------------------------------------

def test_model_step_float32_numpy(torch_cuda, audio):
    """float32 numpy goes through the host float path; float64 numpy keeps the host conversion; both equal step(to_int16(x))"""
    from microwakeword_b200.inference import Model
    base_f, _ = audio
    B = 5
    path = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
    m_f, m_i = Model(path, batch=B), Model(path, batch=B)
    pos = 0
    for n in (480, 480, 16000, 480, 4801):
        x = chunk(base_f, B, pos, n)
        if n == 4801:
            x = x.astype(np.float64)                         # converted by to_int16 inside step, as before
        with np.errstate(invalid="ignore", over="ignore"):
            x_i = to_int16(x)
            same_probs(m_f.step(x), m_i.step(x_i), n)
        pos += n
    same_state(m_f.engine.state_dict(), m_i.engine.state_dict())


# ---- refusals -------------------------------------------------------------------------------------------------------------------

def test_refusals_leave_the_handle_unchanged(torch_cuda, audio):
    """Python refuses float64 and wrong shapes (ValueError, as the device path does); the library refuses too-small output
    buffers, a row pitch below n_samples, NULL audio and the one-model float forms on a K = 2 handle (MwwError)"""
    import ctypes
    from microwakeword_b200.engine import MultiModelEngine, StreamEngine
    torch = torch_cuda
    base_f, _ = audio
    S = 70
    eng = StreamEngine(blob("f32"), n_streams=S)
    eng.predict_clip_host(chunk(base_f, S, 0, 4000))
    multi = MultiModelEngine([blob("f32"), blob("int8")], n_streams=S)
    multi.predict_clip_host(chunk(base_f, S, 0, 4000))
    before = [(e.launch_count, e.frontend_buffered, e.state_dict()) for e in (eng, multi)]
    x = chunk(base_f, S, 4000, 48000)
    steps = eng._steps(48000)

    with np.errstate(invalid="ignore", over="ignore"):
        bads = (x.astype(np.float64), x[:-1], x[None], x[:, :, None], x.astype(np.int32), x.astype(np.float16))
    for e in (eng, multi):
        for bad in bads:
            with pytest.raises(ValueError):
                e.predict_clip_host(bad)
        with pytest.raises(ValueError):
            e.predict_clip_remote(x.ctypes.data, 48000, dtype=np.float64)
    with pytest.raises(_lib.MwwError) as err:
        eng.predict_clip_host(x, out=np.empty((S, steps - 1), np.float32))
    assert err.value.code == -1 and "too small" in str(err.value)
    with pytest.raises(_lib.MwwError) as err:
        multi.predict_clip_host(x, out=[np.empty((S, steps), np.float32), np.empty((S, steps - 1), np.float32)])
    assert err.value.code == -1 and "model 1" in str(err.value)
    d = torch.from_numpy(x).cuda()
    with pytest.raises(_lib.MwwError):
        eng.predict_clip_remote(d.data_ptr(), 48000, tiles=4, out=torch.empty((S, steps - 1), device="cuda"), dtype=np.float32)

    L, got = eng._L, ctypes.c_int(0)
    probs = np.empty((S, 128), np.float32)
    dprobs = torch.empty((S, 128), device="cuda")
    assert L.mww_predict_clip_host_f32(eng._h, x.ctypes.data, 48000, 47999, probs.ctypes.data, 128, ctypes.byref(got)) == -1
    assert L.mww_predict_clip_host_f32(eng._h, None, 48000, 48000, probs.ctypes.data, 128, ctypes.byref(got)) == -1
    assert L.mww_predict_clip_remote_f32(eng._h, d.data_ptr(), 48000, 47999, dprobs.data_ptr(), 128, ctypes.byref(got), 4,
                                         eng._cu_stream()) == -1
    for name, fn in (("mww_predict_clip_host_f32", lambda: L.mww_predict_clip_host_f32(multi._h, x.ctypes.data, 48000, 48000,
                                                                                        probs.ctypes.data, 128, ctypes.byref(got))),
                     ("mww_predict_clip_remote_f32", lambda: L.mww_predict_clip_remote_f32(multi._h, d.data_ptr(), 48000, 48000,
                                                                                            dprobs.data_ptr(), 128, ctypes.byref(got), 4,
                                                                                            multi._cu_stream()))):
        assert fn() == -1, name
        msg = L.mww_last_error(multi._h).decode()
        assert name in msg and "2 models" in msg, (name, msg)
    torch.cuda.synchronize()
    after = [(e.launch_count, e.frontend_buffered, e.state_dict()) for e in (eng, multi)]
    for (l0, b0, s0), (l1, b1, s1) in zip(before, after):
        assert (l0, b0) == (l1, b1)
        same_state(s0, s1)
