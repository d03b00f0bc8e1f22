"""hybrid_ref -- CPU oracle for hybrid models (TEST INFRASTRUCTURE): ctypes front-end of hybrid_ref.c, the [UPSTREAM-RECALL]
restatement of TFLite's hybrid kernels (float graph, int8 weights quantised per channel, input quantised on every invoke).

    hybrid_ref.HybridNet(blob)    -> one stream of a hybrid container: step, state, reset, predict_u16
    hybrid_ref.quantize(x, sym)   -> the hybrid input quantiser on one tensor (codes, scale, zero point)
    hybrid_ref.run_pipeline(...)  -> audio -> features (oracle frontend) -> hybrid probabilities, every stream from reset

The library is compiled on first use (gcc, -ffp-contract=off) into a cache directory outside the tree, keyed by the
source's hash."""

from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "hybrid_ref.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        with open(_SRC, "rb") as f:
            tag = hashlib.sha256(f.read()).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), "mww_hybrid_ref_%d" % os.getuid())
        so = os.path.join(out_dir, "libhybrid_ref_%s.so" % tag)
        if not os.path.exists(so):
            os.makedirs(out_dir, exist_ok=True)
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.run([os.environ.get("CC", "gcc"), "-O3", "-march=x86-64-v3", "-fPIC", "-shared", "-Wall", "-fno-fast-math",
                            "-ffp-contract=off", "-o", tmp, _SRC, "-lm"], check=True)
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, sz, i32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        L.hyref_create.restype = vp
        L.hyref_create.argtypes = [ctypes.c_char_p, sz]
        L.hyref_free.argtypes = [vp]
        L.hyref_reset.argtypes = [vp]
        L.hyref_stride.argtypes = [vp]
        L.hyref_get_state.restype = sz
        L.hyref_get_state.argtypes = [vp, vp, sz]
        L.hyref_step.restype = ctypes.c_float
        L.hyref_step.argtypes = [vp, vp, vp]
        L.hyref_predict_u16.restype = sz
        L.hyref_predict_u16.argtypes = [vp, vp, sz, vp, sz]
        L.hyref_quantize.restype = None
        L.hyref_quantize.argtypes = [i32, vp, i32, vp, vp, vp]
        _lib = L
    return _lib


class HybridNet:
    """One stream of a hybrid MWW container (bytes) on the CPU oracle."""

    def __init__(self, blob: bytes):
        self._L = lib()
        self._h = self._L.hyref_create(blob, len(blob))
        if not self._h:
            raise ValueError("hybrid oracle: malformed container, or no hy/mode tensor")
        self.stride = self._L.hyref_stride(self._h)

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.hyref_free(self._h)
            self._h = None

    def reset(self):
        self._L.hyref_reset(self._h)

    def step(self, x: np.ndarray):
        """one invoke on [stride, 40] float32 rows -> (probability, logit)"""
        x = np.ascontiguousarray(x, np.float32)
        logit = ctypes.c_float(0)
        p = self._L.hyref_step(self._h, x.ctypes.data, ctypes.addressof(logit))
        return np.float32(p), np.float32(logit.value)

    def state(self) -> np.ndarray:
        """ring state in the engine's per-stream layout (StreamEngine.state_dict()["nn"] of one stream)"""
        n = self._L.hyref_get_state(self._h, None, 0)
        out = np.zeros(n, np.float32)
        self._L.hyref_get_state(self._h, out.ctypes.data, n)
        return out

    def predict_u16(self, feat: np.ndarray) -> np.ndarray:
        feat = np.ascontiguousarray(feat, np.uint16)
        probs = np.zeros(feat.shape[0] // max(self.stride, 1) + 1, np.float32)
        n = self._L.hyref_predict_u16(self._h, feat.ctypes.data, feat.shape[0], probs.ctypes.data, probs.size)
        return probs[:n]


def quantize(x: np.ndarray, symmetric: bool = False):
    """the hybrid kernels' input quantiser: float32 tensor -> (int8 codes, scale, zero point)"""
    x = np.ascontiguousarray(x, np.float32).ravel()
    q = np.zeros(x.size, np.int8)
    sc, zp = ctypes.c_float(0), ctypes.c_int32(0)
    lib().hyref_quantize(2 if symmetric else 1, x.ctypes.data, x.size, q.ctypes.data, ctypes.addressof(sc), ctypes.addressof(zp))
    return q, np.float32(sc.value), int(zp.value)


def run_pipeline(blob: bytes, audio: np.ndarray, threads: int = 1):
    """audio int16 [S, N] -> (features uint16 [S, T, 40], probs float32 [S, T // stride]); every stream starts reset"""
    import oracle
    feats, _ = oracle.run_pipeline(None, audio, want_probs=False, threads=threads)
    probs = []
    for f in feats:
        probs.append(HybridNet(blob).predict_u16(f))
    return feats, np.stack(probs) if probs else np.zeros((0, 0), np.float32)
