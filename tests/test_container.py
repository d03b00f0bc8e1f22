"""The model-container parser (microwakeword_b200/csrc/mww_container.cc) on the CPU: the kernel family and geometry it reads
from every kind of container, the weight arena's alignment, and every refusal mww_create reports for a malformed one, with
its code and message."""

import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import tflite_hybrid_writer as HW
from conftest import GOLDEN
from generic_range import GEOMETRIES, SMEM_CAP, boundary_specs, models
from microwakeword_b200 import model_file as MF
from microwakeword_b200 import tflite_file as TF
from oracle import mixednet_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "microwakeword_b200", "csrc")

COMPILED_F32, COMPILED_I8, GENERIC_F32, GENERIC_I8, HYBRID = range(5)
EMODEL, EUNSUPPORTED = -2, -5
MAX_ENTRIES = 256
_lib = None
_BUILD = tempfile.TemporaryDirectory(prefix="mww_container_test_")


def lib():
    global _lib
    if _lib is None:
        # built outside the tree, which may be read-only
        so = os.path.join(_BUILD.name, "libemul_container.so")
        srcs = [os.path.join(HERE, "emul_container.cc"), os.path.join(CSRC, "mww_container.cc")]
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so] + srcs, check=True)
        _lib = ctypes.CDLL(so)
        _lib.emul_parse_container.restype = ctypes.c_int
    return _lib


def parse(blob):
    """(code, message, info dict or None, arena offsets)"""
    info = np.zeros(8, np.int64)
    offsets = np.zeros(MAX_ENTRIES, np.int64)
    msg = ctypes.create_string_buffer(512)
    buf = ctypes.create_string_buffer(bytes(blob), len(blob))
    rc = lib().emul_parse_container(buf, ctypes.c_size_t(len(blob)), ctypes.c_void_p(info.ctypes.data), ctypes.c_void_p(offsets.ctypes.data),
                                    MAX_ENTRIES, msg, len(msg))
    if rc:
        return rc, msg.value.decode(), None, None
    keys = ("kind", "stride", "pend_cap", "state_elems", "macs_per_step", "arena_bytes", "entries", "tc_f16")
    d = dict(zip(keys, (int(v) for v in info)))
    assert d["entries"] <= MAX_ENTRIES
    return rc, "", d, offsets[:d["entries"]]


def golden(kind):
    return MF.load(os.path.join(GOLDEN, "okay_nabu_synth_%s.mww" % kind))


def hybrid_tensors(spec):
    f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    return TF.tensors_from_tflite(HW.write_hybrid_mixednet(f32, lambda op, n: n >= 1024, True))


def check_ok(tensors, kind):
    rc, msg, info, offsets = parse(MF.write_container(tensors))
    assert rc == 0, msg
    arch = MF.Arch.decode(np.asarray(tensors["arch"], np.int32))
    stride = int(tensors["arch"][2])
    assert info["kind"] == kind
    assert (info["stride"], info["pend_cap"]) == (stride, max(stride - 1, 1))
    assert (info["state_elems"], info["macs_per_step"]) == (arch.state_elements, arch.macs_per_step)
    assert len(offsets) > 0 and np.all(offsets % 256 == 0) and np.all(offsets < info["arena_bytes"])
    assert len(set(offsets.tolist())) == len(offsets)
    return info


@pytest.mark.parametrize("kind", ["f32", "int8"])
def test_okay_nabu_runs_on_the_compiled_kernels(kind, monkeypatch):
    monkeypatch.delenv("MWW_FORCE_GENERIC", raising=False)
    info = check_ok(golden(kind), COMPILED_F32 if kind == "f32" else COMPILED_I8)
    assert info["stride"] == 3 and info["pend_cap"] == 2 and info["state_elems"] == 4176 and info["macs_per_step"] == 24800
    monkeypatch.setenv("MWW_FORCE_GENERIC", "1")
    check_ok(golden(kind), GENERIC_F32 if kind == "f32" else GENERIC_I8)


@pytest.mark.parametrize("name", list(GEOMETRIES) + ["boundary"])
def test_generic_range_geometries(name):
    spec = boundary_specs()[SMEM_CAP // 4] if name == "boundary" else GEOMETRIES[name]
    f32, q8 = models(spec)
    check_ok(f32, GENERIC_F32)
    check_ok(q8, GENERIC_I8)


@pytest.mark.parametrize("spec", [R.Spec(), R.Spec(64, 5, 3, (32, 48), ((9, 33), (3,)), head_rows=5)], ids=["okay_nabu", "two_blocks"])
def test_hybrid_container(spec):
    check_ok(hybrid_tensors(spec), HYBRID)


def refusal(tensors_or_blob):
    blob = tensors_or_blob if isinstance(tensors_or_blob, bytes) else MF.write_container(tensors_or_blob)
    rc, msg, _, _ = parse(blob)
    return rc, msg


def without(t, name):
    return {k: v for k, v in t.items() if k != name}


def replaced(t, name, value):
    out = dict(t)
    out[name] = value
    return out


ARCH_MSG = "model container: missing 'arch' tensor or bad magic/version"


def test_refuses_bad_magic_and_truncated_directories():
    blob = MF.write_container(golden("f32"))
    assert refusal(b"XWWB200\0" + blob[8:]) == (EMODEL, ARCH_MSG)
    assert refusal(blob[:8] + (2).to_bytes(4, "little") + blob[12:]) == (EMODEL, ARCH_MSG)      # container version
    assert refusal(blob[:30]) == (EMODEL, ARCH_MSG)                                               # directory cut short
    rc, msg = refusal(blob[:len(blob) // 2])                                                      # tensors cut short
    assert rc == EMODEL and msg.startswith("model container: missing tensor ")


def test_refuses_a_missing_or_malformed_arch():
    t = golden("f32")
    blob = MF.write_container(t)
    assert refusal(blob.replace(b"arch\0", b"arcx\0", 1)) == (EMODEL, ARCH_MSG)                 # no tensor named arch
    assert refusal(replaced(t, "arch", t["arch"].astype(np.float32))) == (EMODEL, ARCH_MSG)
    bad = np.array(t["arch"], np.int32)
    bad[3] = 41                                                                                  # 41 features
    assert refusal(replaced(t, "arch", bad)) == (EMODEL, "model container: malformed 'arch' tensor")
    assert refusal(replaced(t, "arch", bad[:5])) == (EMODEL, "model container: malformed 'arch' tensor")


RANGE_MSG = ("model container: architecture outside the supported range (first_conv_kernel_size >= stride, <= 8 blocks, <= 512 channels, "
             "kernels <= 64 taps, ring buffers of one stream within 200 KB)")


def test_refuses_geometries_outside_the_range():
    assert refusal({"arch": boundary_specs()[SMEM_CAP // 4 + 1].encode()}) == (EUNSUPPORTED, RANGE_MSG)       # 4 bytes over 200 KB
    assert refusal({"arch": R.Spec(513, 5, 3, (64,), ((5,),), head_rows=4).encode()}) == (EUNSUPPORTED, RANGE_MSG)
    assert refusal({"arch": R.Spec(32, 2, 3, (64,), ((5,),), head_rows=4).encode()}) == (EUNSUPPORTED, RANGE_MSG)   # kernel < stride


@pytest.mark.parametrize("kind", ["f32", "int8", "generic_f32", "generic_int8"])
def test_refuses_a_missing_tensor_or_a_wrong_dtype_or_size(kind):
    if kind.startswith("generic"):
        f32, q8 = models(GEOMETRIES["long_stride"])
        t = f32 if kind == "generic_f32" else q8
    else:
        t = golden(kind)
    q = "q/" if "int8" in kind else ""
    w, b = q + "b1/pw/w", q + ("b0/dw/bias" if q else "b0/dw/b")
    assert refusal(without(t, w)) == (EMODEL, "model container: missing tensor " + w)
    assert refusal(without(t, q + "head/w")) == (EMODEL, "model container: missing tensor " + q + "head/w")
    wrong = t[w].astype(np.int16)
    assert refusal(replaced(t, w, wrong)) == (EMODEL, "model container: wrong dtype/size for " + w)
    assert refusal(replaced(t, b, t[b][:-1])) == (EMODEL, "model container: wrong dtype/size for " + b)


@pytest.mark.parametrize("kind", ["int8", "generic_int8"])
def test_refuses_bad_quantisation_parameters(kind):
    t = golden("int8") if kind == "int8" else models(GEOMETRIES["long_stride"])[1]
    assert refusal(without(t, "q/head/bias")) == (EMODEL, "model container: q/head/bias")
    assert refusal(replaced(t, "q/head/shift", np.zeros(2, np.int32))) == (EMODEL, "model container: q/head/shift")
    entries = "12" if kind == "int8" else "4 + 2 * n_blocks"
    msg = "model container: q/scales / q/zps must hold %s entries" % entries
    assert refusal(replaced(t, "q/zps", t["q/zps"][:-1])) == (EMODEL, msg)
    assert refusal(replaced(t, "q/scales", np.append(t["q/scales"], np.float32(1)))) == (EMODEL, msg)


def test_refuses_a_mismatched_hybrid_mode():
    t = hybrid_tensors(R.Spec())
    mode = np.asarray(t["hy/mode"], np.int32)
    mismatch = ("model container: 'hy/mode' does not match the architecture (one entry per first conv, MixConv group, 1x1 conv, head; "
                "0..2)")
    assert refusal(replaced(t, "hy/mode", mode[:-1])) == (EMODEL, mismatch)
    assert refusal(replaced(t, "hy/mode", np.append(mode, np.int32(0)))) == (EMODEL, mismatch)
    assert refusal(replaced(t, "hy/mode", np.where(np.arange(mode.size) == 0, 3, mode).astype(np.int32))) == (EMODEL, mismatch)
    assert refusal(replaced(t, "hy/mode", mode.astype(np.float32))) == (EMODEL, "model container: malformed 'hy/mode'")
    assert refusal(replaced(t, "hy/mode", np.zeros(100, np.int32))) == (EMODEL, "model container: malformed 'hy/mode'")
    assert mode[0] != 0
    assert refusal(without(t, "hy/first_conv/scale")) == (EMODEL, "model container: missing tensor hy/first_conv/scale")


@pytest.mark.gpu
def test_frontend_only_handle_reports_okay_nabu_geometry(torch_cuda):
    from microwakeword_b200.engine import StreamEngine
    info = StreamEngine(None, n_streams=2)._info()
    assert (info.input_feature_slices, info.state_bytes_per_stream, info.macs_per_step, info.is_quantized, info.pending_rows) == (3, 16704, 24800, 0, 0)
