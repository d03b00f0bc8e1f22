"""Build libmww_b200.so in-tree with nvcc for sm_90a (no JIT cache: the .so travels with the repo
snapshot to the GPU box).  `python -m microwakeword_b200.build` or `__graft_entry__.build()`."""

from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libmww_b200.so")
SOURCES = ["mww_capi.cu", "mww_frontend.cu", "mww_nn.cu", "mww_nn_int8.cu", "mww_nn_live.cu", "mww_nn_i8_live.cu", "mww_nn_generic.cu", "mww_nn_tc.cu", "mww_detect.cu", "mww_tables.cc"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-shared",
         "-Xcompiler", "-fPIC", "-cudart", "static"]


STAMP = OUT + ".srchash"


def source_hash() -> str:
    """sha256 over every file of csrc/, include/mww.h and the compiler flags: what the binary was built from.  Content, not
    mtimes -- the tree is copied to the GPU box, where timestamps mean nothing."""
    import hashlib
    h = hashlib.sha256(" ".join(FLAGS).encode())
    deps = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(os.path.dirname(HERE), "include", "mww.h")]
    for d in deps:
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stale() -> bool:
    if not os.path.exists(OUT) or not os.path.exists(STAMP):
        return True
    try:
        return open(STAMP).read().strip() != source_hash()
    except OSError:
        return True


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError("nvcc not found at %s; libmww_b200.so must be prebuilt (there is no CPU fallback)" % NVCC)
    import fcntl
    with open(OUT + ".lock", "w") as lock:               # several ranks may arrive here at once: one builds, the rest wait
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not _stale():
            return OUT
        tmp = OUT + ".tmp.%d" % os.getpid()
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + [os.path.join(CSRC, s) for s in SOURCES]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            if os.path.exists(tmp):
                os.unlink(tmp)
            raise RuntimeError("nvcc failed building libmww_b200.so")
        if verbose:
            sys.stderr.write(res.stderr)
        os.replace(tmp, OUT)                               # a process that has the old file mapped keeps its own copy
        with open(STAMP, "w") as f:
            f.write(source_hash() + "\n")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
