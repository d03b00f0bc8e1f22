"""ctypes front-end of tests/host_emul/emul_hybrid.cc -- TEST INFRASTRUCTURE: the hybrid (fp32 graph, int8-weight ops)
phase functions of microwakeword_b200/csrc/mww_nn_generic.cuh executed thread by thread on the CPU."""

import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "microwakeword_b200", "csrc")
SO = os.path.join(HERE, "_build", "libemul_hybrid.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "emul_hybrid.cc")
        deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
        if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
            os.makedirs(os.path.dirname(SO), exist_ok=True)
            # -ffp-contract=off: the phase functions' float operations are the oracle's, one rounding each
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", SO, src], check=True)
        L = ctypes.CDLL(SO)
        L.emul_hy_run.restype = ctypes.c_int
        L.emul_hy_thread_order.restype = None
        _lib = L
    return _lib


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def quantize(x, symmetric=False):
    """the device formulation of the hybrid input quantiser -> (int8 codes, scale, zero point)"""
    x = np.ascontiguousarray(x, np.float32).ravel()
    q = np.zeros(x.size, np.int8)
    sc, zp = ctypes.c_float(0), ctypes.c_int32(0)
    lib().emul_hy_quantize(2 if symmetric else 1, _p(x), x.size, _p(q), ctypes.byref(sc), ctypes.byref(zp))
    return q, np.float32(sc.value), int(zp.value)


class GenHybrid:
    """Hybrid MixedNet of any architecture stepped with the generic hybrid kernel's phase functions; `tensors` = container"""

    def __init__(self, tensors, n_streams):
        from host_emul import emul
        self.arch = np.ascontiguousarray(tensors["arch"], np.int32)
        self.modes = np.ascontiguousarray(tensors["hy/mode"], np.int32)
        info = emul.gen_arch_info(self.arch)
        assert info["rc"] == 0, info
        self.info = info
        nb = int(self.arch[4])
        names = ["first_conv/w"]
        for i in range(nb):
            names += ["b%d/dw/w" % i, "b%d/dw/b" % i, "b%d/pw/w" % i, "b%d/pw/b" % i]
        names += ["head/w", "head/b"]
        self.f = [np.ascontiguousarray(tensors[n], np.float32) for n in names]
        self.wf = (ctypes.c_void_p * len(self.f))(*[a.ctypes.data for a in self.f])
        hnames = ["hy/first_conv/w", "hy/first_conv/scale"]
        for i in range(nb):
            hnames += ["hy/b%d/dw/w" % i, "hy/b%d/dw/scale" % i, "hy/b%d/pw/w" % i, "hy/b%d/pw/scale" % i]
        hnames += ["hy/head/w", "hy/head/scale"]
        self.h = [np.ascontiguousarray(tensors[n]) if n in tensors else None for n in hnames]
        self.wh = (ctypes.c_void_p * len(self.h))(*[(a.ctypes.data if a is not None else None) for a in self.h])
        self.state = np.zeros((n_streams, info["state_elems"]), np.float32)
        self.pend = np.zeros((n_streams, info["pend_cap"] * 40), np.float32)
        self.n_pend = 0
        self.stride = info["stride"]
        self.sm_bytes = 0

    def infer(self, rows):
        rows = np.ascontiguousarray(rows)
        S, n_rows = rows.shape[:2]
        rt = {np.dtype(np.uint16): 0, np.dtype(np.float32): 1}[rows.dtype]
        probs = np.zeros((S, (self.n_pend + n_rows) // self.stride + 1), np.float32)
        smb = ctypes.c_longlong(0)
        n = lib().emul_hy_run(_p(self.arch), self.arch.size, _p(self.modes), self.modes.size, self.wf, self.wh, _p(self.state), _p(self.pend),
                              self.n_pend, _p(rows), n_rows, rt, S, _p(probs), probs.shape[1], ctypes.byref(smb))
        assert n >= 0, n
        self.sm_bytes = smb.value
        self.n_pend = (self.n_pend + n_rows) % self.stride
        return probs[:, :n]
