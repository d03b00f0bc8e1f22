"""Each model of a multi-model handle on its own streams (mww_create_multi_streams), the parts that need no GPU: the tile
planner and the gather / remap / id-translation index math of microwakeword_b200/csrc/mww_streams.h (built with g++ in a
temporary directory, since the tree may be read-only) against brute force and numpy fancy indexing, MultiModelEngine's
argument checks, and the instruction SASS of every kernel the library had before stream sets, which must not change."""

import ctypes
import hashlib
import json
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "microwakeword_b200", "csrc")
_BUILD = tempfile.TemporaryDirectory(prefix="mww_streams_test_")
_emul = None


def emul():
    global _emul
    if _emul is None:
        so = os.path.join(_BUILD.name, "libemul_streams.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_streams.cc")], check=True)
        _emul = ctypes.CDLL(so)
    return _emul


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def _random_set(rng, S, kind):
    if kind == "empty":
        return np.zeros(0, np.int32)
    if kind == "all":
        return np.arange(S, dtype=np.int32)
    if kind == "last":
        return np.array([S - 1], np.int32)
    if kind == "block":
        a = int(rng.integers(0, S))
        return np.arange(a, int(rng.integers(a, S)) + 1, dtype=np.int32)
    if kind == "interleaved":
        step = int(rng.integers(2, 6))
        return np.arange(int(rng.integers(0, step)), S, step, dtype=np.int32)
    return np.flatnonzero(rng.random(S) < rng.random()).astype(np.int32)


@pytest.mark.parametrize("seed", range(40))
def test_tile_planner_agrees_with_brute_force(seed):
    rng = np.random.default_rng(seed)
    S = int(rng.choice([1, 2, 7, 70, 829, 4096]))
    L = emul()
    for kind in ("empty", "all", "last", "block", "interleaved", "random", "random"):
        ids = _random_set(rng, S, kind)
        for tile in sorted({1, 3, int(rng.integers(1, S + 1)), S}):
            T = -(-S // tile)
            a, b, cons = np.zeros(T, np.int32), np.zeros(T, np.int32), np.zeros(T, np.int32)
            assert L.emul_tile_plan(_p(ids), ids.size, S, tile, _p(a), _p(b), _p(cons)) == T
            for t in range(T):
                first, last = t * tile, min(t * tile + tile, S)
                members = [j for j, s in enumerate(ids) if first <= s < last]
                want_a = members[0] if members else int(np.searchsorted(ids, first))
                assert (a[t], b[t]) == (want_a, want_a + len(members)), (kind, tile, t)
                sel = ids[a[t]:b[t]]
                assert bool(cons[t]) == (sel.size == 0 or np.array_equal(sel, np.arange(sel[0], sel[0] + sel.size))), (kind, tile, t)
            if kind in ("all", "block", "last", "empty"):
                assert cons.all()                          # consecutive members never need the gather
            assert b[-1] - a[0] == ids.size


def test_stream_set_validation():
    L = emul()
    for ids, S, ok in (([], 5, True), ([0, 1, 4], 5, True), ([4], 5, True), ([1, 1], 5, False), ([2, 1], 5, False),
                       ([-1], 5, False), ([5], 5, False)):
        a = np.asarray(ids, np.int32)
        assert bool(L.emul_valid_stream_set(_p(a), a.size, S)) == ok, ids


@pytest.mark.parametrize("F", [1, 3, 298])
def test_gather_index_math_is_fancy_indexing(F):
    rng = np.random.default_rng(F)
    S, tile = 300, 128
    feat = rng.integers(0, 2048, (S, F, 40)).astype(np.uint16)
    ids = np.flatnonzero(rng.random(S) < 0.4).astype(np.int32)
    L = emul()
    for first in range(0, S, tile):
        last = min(first + tile, S)
        a, b = int(np.searchsorted(ids, first)), int(np.searchsorted(ids, last))
        rows = np.ascontiguousarray(feat[first:last])
        out = np.zeros((b - a, F, 40), np.uint16)
        L.emul_gather(_p(rows), _p(ids), a, first, b - a, ctypes.c_longlong(F * 80 // 16), _p(out))
        assert np.array_equal(out, feat[ids[a:b]])
        assert out.strides[0] % 16 == 0                      # the int8 and wgmma kernels' row alignment


def test_remap_and_id_translation_are_fancy_indexing():
    rng = np.random.default_rng(7)
    S, W = 500, 13
    for _ in range(20):
        old = np.flatnonzero(rng.random(S) < rng.random()).astype(np.int32)
        new = np.flatnonzero(rng.random(S) < rng.random()).astype(np.int32)
        inv = np.full(S, -1, np.int32)
        inv[old] = np.arange(old.size, dtype=np.int32)
        old_index = inv[new]
        src = rng.integers(0, 1 << 32, (max(old.size, 1), W), dtype=np.uint64).astype(np.uint32)
        dst = np.full((new.size, W), 0xDEADBEEF, np.uint32)
        L = emul()
        L.emul_remap(_p(dst), _p(src), ctypes.c_longlong(W), _p(old_index), new.size)
        kept = old_index >= 0
        assert np.array_equal(dst[kept], src[old_index[kept]])
        assert (dst[~kept] == 0xDEADBEEF).all()
        ids = rng.integers(-3, S + 3, 200).astype(np.int32)
        out = np.zeros_like(ids)
        L.emul_compact_ids(_p(out), _p(ids), ids.size, _p(inv), S)
        inside = (ids >= 0) & (ids < S)
        assert np.array_equal(out[inside], inv[ids[inside]]) and (out[~inside] == -1).all()


def test_engine_refuses_bad_stream_sets_before_the_library():
    from microwakeword_b200.engine import MultiModelEngine
    f32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
    i8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
    for streams in ([[2, 1], None], [[0, 0], None], [[0, 8], None], [[-1], None], [None], [None, None, None], [[[0, 1]], None]):
        with pytest.raises(ValueError):
            MultiModelEngine([f32, i8], n_streams=8, streams=streams)


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    from microwakeword_b200 import _lib
    from microwakeword_b200.engine import MultiModelEngine
    f32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
    with pytest.raises(_lib.MwwError) as e:
        MultiModelEngine([f32, f32], n_streams=8, streams=[[0, 2, 4], None])
    assert e.value.code == -3 and "no CUDA device" in str(e.value)


# ---- the kernels that existed before stream sets compile to the same instructions ------------------------------------
SASS_GOLDEN = os.path.join(GOLDEN, "sass_kernels_before_stream_sets.json")


def sass_functions(so):
    """{kernel name: sha256 of its instruction SASS} of a library, from cuobjdump -sass"""
    cuobjdump = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", so], capture_output=True, text=True, check=True).stdout
    # names in anonymous namespaces carry hashes of the build path: keep the file name only
    text = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_\d+_(\w+?_cu)_[0-9a-f]{8}", r"_GLOBAL__N__\1", text)
    out, name, body = {}, None, []
    for line in text.splitlines() + ["Function : <end>"]:
        m = re.match(r"\s*Function : (\S+)", line)
        if m or line.startswith("Fatbin") or "....." in line:
            if name is not None:
                out[name] = hashlib.sha256("\n".join(body).encode()).hexdigest()
            name, body = (m.group(1) if m else None), []
        elif name is not None and line.strip():
            body.append(line.strip())
    out.pop("<end>", None)
    return out


def test_existing_kernels_sass_unchanged():
    from microwakeword_b200 import _lib, build
    _lib.lib()                                               # builds the library if needed
    if not os.path.exists(os.path.join(os.path.dirname(build.NVCC), "cuobjdump")):
        pytest.skip("cuobjdump is not installed next to nvcc")
    got = sass_functions(build.OUT)
    want = json.load(open(SASS_GOLDEN))
    assert len(want) >= 30
    changed = sorted(k for k in want if got.get(k) != want[k])
    assert not changed, changed
