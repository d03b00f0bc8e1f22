"""Loader for the reference's streaming ``.tflite`` models (SURVEY.md section 8 f-2).

``microwakeword.inference.Model(tflite_model_path)`` hands the file to ``tf.lite.Interpreter``
(inference.py:36-45).  Neither TensorFlow nor the ``flatbuffers`` module exists in this build, so this
module reads the TFL3 flatbuffer directly (wire format only: vtables, vectors, unions) and *recognises*
the one graph family the hot path implements -- the internal-state streaming MixedNet that
``utils.convert_saved_model_to_tflite`` (utils.py:289-348) emits for ``mixednet.model``
(mixednet.py:278-386) -- turning it into the tensor dictionary of ``model_file`` (the ``.mww``
container the C-ABI consumes).  It is a recogniser, not an interpreter: anything that does not have the
expected structure (ring-buffer variable -> CONCATENATION -> conv, MixConv SPLIT_V / DEPTHWISE_CONV_2D
groups, 1x1 CONV_2D + fused RELU, FULLY_CONNECTED + LOGISTIC) raises ``TfliteError`` naming the
operator, so an unsupported model fails loudly at ``Model(path)`` instead of producing numbers.

PARITY UNPINNED: no ``.tflite`` file produced by TensorFlow exists in this environment
(SURVEY.md 8c).  The schema field numbers and builtin operator codes below are restated from the
public ``tensorflow/lite/schema/schema.fbs`` (v3); the loader is validated against files written by
``tests/tflite_writer.py`` and against an op-by-op executor of the same bytes kept with the test infrastructure.
"""

from __future__ import annotations

import struct

import numpy as np

from . import model_file as MF

FILE_IDENTIFIER = b"TFL3"


class TfliteError(ValueError):
    pass


# ---------------------------------------------------------------------------------------------
# flatbuffer wire format (read side)

class Table:
    """One flatbuffer table: field lookup through its vtable."""

    __slots__ = ("buf", "pos", "_vt", "_vt_len")

    def __init__(self, buf: bytes, pos: int):
        if pos < 0 or pos + 4 > len(buf):
            raise TfliteError("flatbuffer table offset %d outside the file" % pos)
        self.buf, self.pos = buf, pos
        self._vt = pos - struct.unpack_from("<i", buf, pos)[0]
        if self._vt < 0 or self._vt + 4 > len(buf):
            raise TfliteError("flatbuffer vtable offset outside the file")
        self._vt_len = struct.unpack_from("<H", buf, self._vt)[0]

    def _field(self, idx: int) -> int:
        o = 4 + 2 * idx
        if o + 2 > self._vt_len:
            return 0
        off = struct.unpack_from("<H", self.buf, self._vt + o)[0]
        return self.pos + off if off else 0

    def scalar(self, idx: int, fmt: str, default=0):
        p = self._field(idx)
        return struct.unpack_from("<" + fmt, self.buf, p)[0] if p else default

    def _indirect(self, idx: int) -> int:
        p = self._field(idx)
        return p + struct.unpack_from("<I", self.buf, p)[0] if p else 0

    def table(self, idx: int):
        p = self._indirect(idx)
        return Table(self.buf, p) if p else None

    def string(self, idx: int) -> str:
        p = self._indirect(idx)
        if not p:
            return ""
        n = struct.unpack_from("<I", self.buf, p)[0]
        if p + 4 + n > len(self.buf):
            raise TfliteError("flatbuffer string runs past the end of the file")
        return bytes(self.buf[p + 4:p + 4 + n]).decode("utf-8", "replace")

    def vector(self, idx: int, dtype) -> np.ndarray:
        p = self._indirect(idx)
        if not p:
            return np.zeros(0, dtype)
        n = struct.unpack_from("<I", self.buf, p)[0]
        dt = np.dtype(dtype).newbyteorder("<")
        if p + 4 + n * dt.itemsize > len(self.buf):
            raise TfliteError("flatbuffer vector runs past the end of the file")
        return np.frombuffer(self.buf, dt, n, p + 4)

    def tables(self, idx: int) -> list:
        p = self._indirect(idx)
        if not p:
            return []
        n = struct.unpack_from("<I", self.buf, p)[0]
        if p + 4 + 4 * n > len(self.buf):
            raise TfliteError("flatbuffer vector of tables runs past the end of the file")
        out = []
        for i in range(n):
            e = p + 4 + 4 * i
            out.append(Table(self.buf, e + struct.unpack_from("<I", self.buf, e)[0]))
        return out


# ---------------------------------------------------------------------------------------------
# TFL3 schema subset (tensorflow/lite/schema/schema.fbs; field ids in declaration order)

TENSOR_TYPES = {0: np.float32, 2: np.int32, 3: np.uint8, 4: np.int64, 7: np.int16, 9: np.int8}
TYPE_RESOURCE = 13

OP_CONCATENATION, OP_CONV_2D, OP_DEPTHWISE_CONV_2D, OP_FULLY_CONNECTED, OP_LOGISTIC, OP_RELU = 2, 3, 4, 9, 14, 19
OP_RESHAPE, OP_SQUEEZE, OP_STRIDED_SLICE, OP_SPLIT, OP_EXPAND_DIMS, OP_SPLIT_V, OP_QUANTIZE = 22, 43, 45, 49, 70, 102, 114
OP_CALL_ONCE, OP_VAR_HANDLE, OP_READ_VARIABLE, OP_ASSIGN_VARIABLE = 129, 142, 143, 144
OP_NAMES = {2: "CONCATENATION", 3: "CONV_2D", 4: "DEPTHWISE_CONV_2D", 9: "FULLY_CONNECTED", 14: "LOGISTIC", 19: "RELU",
            22: "RESHAPE", 43: "SQUEEZE", 45: "STRIDED_SLICE", 49: "SPLIT", 70: "EXPAND_DIMS", 102: "SPLIT_V", 114: "QUANTIZE",
            129: "CALL_ONCE", 142: "VAR_HANDLE", 143: "READ_VARIABLE", 144: "ASSIGN_VARIABLE"}
PADDING_VALID = 1
ACT_NONE, ACT_RELU = 0, 1


class Tensor:
    def __init__(self, t: Table, buffers: list, index: int):
        self.index = index
        self.shape = tuple(int(x) for x in t.vector(0, np.int32))
        self.type = t.scalar(1, "b")
        self.buffer = t.scalar(2, "I")
        self.name = t.string(3)
        q = t.table(4)
        self.scale = q.vector(2, np.float32).copy() if q else np.zeros(0, np.float32)
        self.zero_point = q.vector(3, np.int64).copy() if q else np.zeros(0, np.int64)
        self.quantized_dimension = q.scalar(6, "i") if q else 0
        self.is_variable = bool(t.scalar(5, "B"))
        self._buffers = buffers

    @property
    def dtype(self):
        if self.type not in TENSOR_TYPES:
            raise TfliteError("tensor %r has unsupported type code %d" % (self.name, self.type))
        return np.dtype(TENSOR_TYPES[self.type])

    @property
    def is_constant(self) -> bool:
        return 0 < self.buffer < len(self._buffers) and self._buffers[self.buffer].size > 0

    def data(self) -> np.ndarray:
        if not self.is_constant:
            raise TfliteError("tensor %r is not a constant" % self.name)
        raw = self._buffers[self.buffer]
        n = int(np.prod(self.shape)) if self.shape else 1
        if raw.size != n * self.dtype.itemsize:
            raise TfliteError("tensor %r: buffer holds %d bytes, shape %s needs %d" % (self.name, raw.size, self.shape, n * self.dtype.itemsize))
        return np.frombuffer(raw.tobytes(), self.dtype.newbyteorder("<")).reshape(self.shape).astype(self.dtype)

    def per_tensor_q(self):
        if self.scale.size != 1 or self.zero_point.size != 1:
            raise TfliteError("tensor %r needs per-tensor quantisation parameters (has %d scales)" % (self.name, self.scale.size))
        return np.float32(self.scale[0]), int(self.zero_point[0])


class Operator:
    def __init__(self, t: Table, codes: list, index: int):
        self.index = index
        self.code = codes[t.scalar(0, "I")]
        self.inputs = [int(x) for x in t.vector(1, np.int32)]
        self.outputs = [int(x) for x in t.vector(2, np.int32)]
        self.options = t.table(4)

    @property
    def name(self):
        return OP_NAMES.get(self.code, "builtin#%d" % self.code)

    def opt(self, idx, fmt, default=0):
        return self.options.scalar(idx, fmt, default) if self.options is not None else default


class Graph:
    """Subgraph 0 of a TFL3 file plus (when present) the variable initialisers of the CALL_ONCE subgraph."""

    def __init__(self, blob: bytes):
        blob = bytes(blob)
        if len(blob) < 16 or blob[4:8] != FILE_IDENTIFIER:
            raise TfliteError("not a TFL3 flatbuffer (file identifier %r)" % blob[4:8])
        root = Table(blob, struct.unpack_from("<I", blob, 0)[0])
        self.version = root.scalar(0, "I")
        codes = []
        for oc in root.tables(1):
            dep, new = oc.scalar(0, "b"), oc.scalar(3, "i")
            codes.append(new if new else dep)                    # builtin_code supersedes the deprecated byte field when set
        self.buffers = [b.vector(0, np.uint8) for b in root.tables(4)]
        subgraphs = root.tables(2)
        if not subgraphs:
            raise TfliteError("model has no subgraph")
        self.subgraphs = []
        for sg in subgraphs:
            tensors = [Tensor(t, self.buffers, i) for i, t in enumerate(sg.tables(0))]
            ops = [Operator(o, codes, i) for i, o in enumerate(sg.tables(3))]
            self.subgraphs.append((tensors, ops, [int(x) for x in sg.vector(1, np.int32)], [int(x) for x in sg.vector(2, np.int32)]))
        self.tensors, self.ops, self.inputs, self.outputs = self.subgraphs[0]
        self.producer = {}
        for op in self.ops:
            for o in op.outputs:
                self.producer[o] = op
        self.consumers = {}
        for op in self.ops:
            for i in op.inputs:
                if i >= 0:
                    self.consumers.setdefault(i, []).append(op)


# ---------------------------------------------------------------------------------------------
# recogniser

def quantize_multiplier(real: float):
    """TFLite ``QuantizeMultiplier``: real = M0 * 2^(shift-31) with M0 in [2^30, 2^31)."""
    if real == 0.0:
        return 0, 0
    m, e = np.frexp(np.float64(real))
    q = int(np.round(m * (1 << 31)))
    if q == (1 << 31):
        q //= 2
        e += 1
    if e < -31:
        return 0, 0
    return int(q), int(e)


def logistic_lut(in_scale, in_zp, out_zp=-128) -> np.ndarray:
    """The 256-entry table the builtin int8 LOGISTIC kernel populates in float (output scale 1/256)."""
    lut = np.zeros(256, np.int8)
    for v in range(-128, 128):
        x = np.float32(in_scale) * np.float32(v - in_zp)
        y = np.float32(1.0) / (np.float32(1.0) + np.exp(-x, dtype=np.float32))
        r = np.round(np.float32(y * np.float32(256.0)))
        lut[v & 0xFF] = np.int8(np.clip(int(r) + out_zp, -128, 127))
    return lut


_PASS_THROUGH = (OP_RESHAPE, OP_SQUEEZE, OP_EXPAND_DIMS)


class _Recogniser:
    def __init__(self, g: Graph):
        self.g = g

    def fail(self, op, msg):
        raise TfliteError("unsupported streaming graph at operator %d (%s): %s" % (op.index, op.name, msg) if op is not None
                          else "unsupported streaming graph: " + msg)

    def t(self, idx):
        return self.g.tensors[idx]

    def ring_memory(self, op, tensor_idx, rows_new):
        """tensor_idx must be CONCATENATION(axis=1)(READ_VARIABLE ring, new rows): return (ring_rows, new-rows tensor index)."""
        c = self.g.producer.get(tensor_idx)
        if c is None or c.code != OP_CONCATENATION or len(c.inputs) != 2:
            self.fail(op, "input is not the CONCATENATION of a ring-buffer variable with the new rows (stream.py:586-590)")
        axis = c.opt(0, "i")
        if axis not in (1, -3):
            self.fail(c, "ring concatenation along axis %d, expected the time axis 1" % axis)
        rd = self.g.producer.get(c.inputs[0])
        if rd is None or rd.code != OP_READ_VARIABLE:
            self.fail(c, "first concatenation input is not a READ_VARIABLE")
        ring, new = self.t(c.inputs[0]), self.t(c.inputs[1])
        mem = self.t(tensor_idx)
        if len(mem.shape) != 4 or mem.shape[0] != 1 or mem.shape[2] != 1 or ring.shape[1] + new.shape[1] != mem.shape[1]:
            self.fail(c, "ring memory shape %s is not [1, ring+new, 1, C]" % (mem.shape,))
        if rows_new is not None and new.shape[1] != rows_new:
            self.fail(c, "%d new rows per step, expected %d" % (new.shape[1], rows_new))
        # the same memory tensor must feed the state update: STRIDED_SLICE (last `ring` rows) -> ASSIGN_VARIABLE
        ok = False
        for s in self.g.consumers.get(tensor_idx, []):
            if s.code == OP_STRIDED_SLICE and self.t(s.outputs[0]).shape == ring.shape:
                ok = ok or any(a.code == OP_ASSIGN_VARIABLE for a in self.g.consumers.get(s.outputs[0], []))
        if not ok:
            self.fail(c, "ring memory is never written back (STRIDED_SLICE -> ASSIGN_VARIABLE missing)")
        if ring.scale.size and (ring.scale.size != mem.scale.size or ring.scale[0] != mem.scale[0] or ring.zero_point[0] != mem.zero_point[0]
                                or new.scale[0] != mem.scale[0] or new.zero_point[0] != mem.zero_point[0]):
            self.fail(c, "ring variable and its input do not share quantisation parameters (utils.py:333)")
        return ring.shape[1], c.inputs[1]

    def skip_back(self, idx, codes=_PASS_THROUGH):
        """walk producers backwards through shape-only ops"""
        while True:
            p = self.g.producer.get(idx)
            if p is None or p.code not in codes:
                return idx
            idx = p.inputs[0]

    def conv_act(self, op, act_field):
        """fused activation, or a stand-alone RELU directly after; returns (is_relu, output tensor index)"""
        act = op.opt(act_field, "b")
        out = op.outputs[0]
        if act == ACT_RELU:
            return True, out
        if act != ACT_NONE:
            self.fail(op, "fused activation %d (only NONE / RELU occur in mixednet.py)" % act)
        cons = self.g.consumers.get(out, [])
        if len(cons) == 1 and cons[0].code == OP_RELU:
            return True, cons[0].outputs[0]
        return False, out

    def run(self) -> dict:
        g = self.g
        if len(g.inputs) != 1 or len(g.outputs) != 1:
            self.fail(None, "expected one input and one output tensor (utils.py:218-222)")
        tin, tout = self.t(g.inputs[0]), self.t(g.outputs[0])
        if int(np.prod(tin.shape)) % MF.NUM_FEATURES or tin.shape[-1] != MF.NUM_FEATURES:
            self.fail(None, "input shape %s is not [1, stride, 40] (modes.py:62-63)" % (tin.shape,))
        stride = int(np.prod(tin.shape)) // MF.NUM_FEATURES
        quantized = tin.dtype == np.int8
        if not quantized and tin.dtype != np.float32:
            self.fail(None, "input dtype %s (int8 or float32 expected, inference.py:99-111)" % tin.dtype)

        compute = [op for op in g.ops if op.code in (OP_CONV_2D, OP_DEPTHWISE_CONV_2D, OP_FULLY_CONNECTED, OP_LOGISTIC)]
        other = [op for op in g.ops if op.code not in OP_NAMES]
        if other:
            self.fail(other[0], "operator outside the streaming MixedNet op set")
        if len(compute) < 4 or compute[0].code != OP_CONV_2D or compute[-1].code != OP_LOGISTIC or compute[-2].code != OP_FULLY_CONNECTED:
            self.fail(None, "expected CONV_2D ... FULLY_CONNECTED, LOGISTIC (mixednet.py:317-384); pooled / attention heads are not supported")

        out = {}
        scales, zps = [], []

        def act_q(tensor):
            if quantized:
                s, z = tensor.per_tensor_q()
                scales.append(s)
                zps.append(z)

        def weights_q(prefix, w_t, w_arr, bias_t, n_out, s_in, s_out):
            """int8 layer tensors in the container's naming; w_arr already in container layout"""
            if w_t.dtype != np.int8:
                self.fail(None, "%s: weights are %s, expected int8" % (prefix, w_t.dtype))
            if np.any(w_t.zero_point != 0):
                self.fail(None, "%s: weight zero points must be 0 (symmetric per-channel quantisation)" % prefix)
            sw = w_t.scale.astype(np.float32)
            if sw.size == 1:
                sw = np.repeat(sw, n_out)
            if sw.size != n_out:
                self.fail(None, "%s: %d weight scales for %d output channels" % (prefix, sw.size, n_out))
            if bias_t is None:
                bias = np.zeros(n_out, np.int32)
            else:
                if bias_t.dtype != np.int32:
                    self.fail(None, "%s: bias is %s, expected int32" % (prefix, bias_t.dtype))
                bias = bias_t.data().reshape(-1).astype(np.int32)
            ms = [quantize_multiplier(np.float64(s_in) * np.float64(s) / np.float64(s_out)) for s in sw]
            out["q/" + prefix + "/w"] = np.ascontiguousarray(w_arr.astype(np.int8))
            out["q/" + prefix + "/bias"] = bias
            out["q/" + prefix + "/mult"] = np.asarray([m for m, _ in ms], np.int32)
            out["q/" + prefix + "/shift"] = np.asarray([s for _, s in ms], np.int32)

        def bias_of(op, n, slot=2):
            if len(op.inputs) <= slot or op.inputs[slot] < 0:
                return None
            b = self.t(op.inputs[slot])
            if int(np.prod(b.shape)) != n:
                self.fail(op, "bias has %s elements, expected %d" % (b.shape, n))
            return b

        # float graph: every weight tensor is float32, or -- dynamic-range quantisation (utils.py:328 without a representative
        # dataset) -- symmetric int8 with one float scale per output channel, executed by TFLite's hybrid kernels.  Decided per
        # op from the file.  Returns (float32 values in the file's layout, int8 codes or None, scales or None).
        hy = {}
        modes = []

        def float_weights(op, w_t, n_out, qdim, bias_t):
            if w_t.dtype == np.float32:
                return w_t.data().astype(np.float32), None, None
            if w_t.dtype != np.int8:
                self.fail(op, "weights are %s in a float graph (float32, or int8 with per-channel scales)" % w_t.dtype)
            if w_t.scale.size != n_out or (w_t.scale.size > 1 and w_t.quantized_dimension != qdim):
                self.fail(op, "int8 weights in a float graph need one scale per output channel on dimension %d; have %d scale(s) for %d "
                              "channels on dimension %d" % (qdim, w_t.scale.size, n_out, w_t.quantized_dimension))
            if w_t.zero_point.size not in (1, n_out) or np.any(w_t.zero_point != 0):
                self.fail(op, "int8 weights in a float graph must have zero points 0 (symmetric quantisation)")
            if bias_t is not None and bias_t.dtype != np.float32:
                self.fail(op, "hybrid op with a %s bias, expected float32" % bias_t.dtype)
            codes = w_t.data()
            s = w_t.scale.astype(np.float32)
            shape = [1] * codes.ndim
            shape[qdim] = n_out
            return (codes.astype(np.float32) * s.reshape(shape)).astype(np.float32), codes, s

        # ---- first conv: Stream(Conv2D(k x 1, strides=(stride, 1), valid, no bias)) + ReLU (mixednet.py:317-331)
        c0 = compute[0]
        w_t = self.t(c0.inputs[1])
        if len(w_t.shape) != 4 or w_t.shape[2] != 1 or w_t.shape[3] != MF.NUM_FEATURES:
            self.fail(c0, "filter shape %s is not [filters, k, 1, 40]" % (w_t.shape,))
        f0, k0 = w_t.shape[0], w_t.shape[1]
        if c0.opt(0, "b") != PADDING_VALID or c0.opt(2, "i", 1) != stride or c0.opt(5, "i", 1) != 1:
            self.fail(c0, "first conv must be VALID with stride_h == %d and no dilation" % stride)
        mem0 = self.skip_back(c0.inputs[0])
        if self.t(mem0).shape != (1, k0, 1, MF.NUM_FEATURES):
            self.fail(c0, "input %s is not one kernel window [1, %d, 1, 40]" % (self.t(mem0).shape, k0))
        ring0, new0 = self.ring_memory(c0, mem0, stride)
        if ring0 != max(0, k0 - 1 - (stride - 1)):
            self.fail(c0, "ring of %d rows, stream.py:253-255 gives %d" % (ring0, max(0, k0 - 1 - (stride - 1))))
        if self.skip_back(new0) != g.inputs[0]:
            self.fail(c0, "first conv does not read the model input")
        relu, cur = self.conv_act(c0, 3)
        if not relu:
            self.fail(c0, "first conv has no ReLU (mixednet.py:331)")
        act_q(tin)
        act_q(self.t(cur))
        w0 = np.transpose(w_t.data()[:, :, 0, :], (1, 2, 0))               # [k, 40, filters]
        b0 = bias_of(c0, f0)
        if quantized:
            weights_q("first_conv", w_t, w0, b0, f0, scales[0], scales[1])
        else:
            if b0 is not None and np.any(b0.data() != 0):
                self.fail(c0, "first conv carries a non-zero bias; mixednet.py:323 builds it with use_bias=False")
            wf, codes, s = float_weights(c0, w_t, f0, 0, b0)
            out["first_conv/w"] = np.ascontiguousarray(np.transpose(wf[:, :, 0, :], (1, 2, 0)))
            modes.append(MF.HYBRID_FLOAT if codes is None else MF.HYBRID_ASYMMETRIC)
            if codes is not None:
                hy["hy/first_conv/w"] = np.ascontiguousarray(np.transpose(codes[:, :, 0, :], (1, 2, 0)))
                hy["hy/first_conv/scale"] = s

        # ---- MixConv blocks (mixednet.py:341-360)
        pw_filters, ksizes = [], []
        i = 1
        cin = f0
        while compute[i].code != OP_FULLY_CONNECTED:
            dws = []
            while compute[i].code == OP_DEPTHWISE_CONV_2D:
                dws.append(compute[i])
                i += 1
            pw = compute[i]
            i += 1
            if pw.code != OP_CONV_2D:
                self.fail(pw, "expected DEPTHWISE_CONV_2D group(s) followed by a 1x1 CONV_2D")
            b = len(pw_filters)
            if not dws:
                # A block whose largest MixConv kernel is 1 has NO MixConv layer in the reference graph (mixednet.py:346-348): the
                # 1x1 conv reads the previous activation directly.  The container keeps one uniform block structure, so the block
                # gets the exact identity as its depthwise stage (tap 1, bias 0; int8: weight 1 at scale 1, multiplier 1.0, the
                # previous tensor's quantisation on both sides).
                pf = self.t(pw.inputs[1])
                if len(pf.shape) != 4 or pf.shape[1:] != (1, 1, cin):
                    self.fail(pw, "filter shape %s is not [filters, 1, 1, %d]" % (pf.shape, cin))
                if pw.inputs[0] != cur:
                    self.fail(pw, "1x1 conv of a block without MixConv does not read the previous layer's output")
                if pw.opt(1, "i", 1) != 1 or pw.opt(2, "i", 1) != 1:
                    self.fail(pw, "1x1 conv with a stride")
                relu, nxt = self.conv_act(pw, 3)
                if not relu:
                    self.fail(pw, "1x1 conv without ReLU (mixednet.py:359)")
                cout = pf.shape[0]
                pw_w = pf.data()[:, 0, 0, :].T
                pb = bias_of(pw, cout)
                if quantized:                                                       # "depthwise output" = the previous tensor itself
                    scales.append(scales[-1])
                    zps.append(zps[-1])
                act_q(self.t(nxt))
                if quantized:
                    m1, s1 = quantize_multiplier(1.0)
                    out["q/b%d/dw/w" % b] = np.ones((1, cin), np.int8)
                    out["q/b%d/dw/bias" % b] = np.zeros(cin, np.int32)
                    out["q/b%d/dw/mult" % b] = np.full(cin, m1, np.int32)
                    out["q/b%d/dw/shift" % b] = np.full(cin, s1, np.int32)
                    weights_q("b%d/pw" % b, pf, pw_w, pb, cout, scales[-2], scales[-1])
                else:
                    wf, codes, s = float_weights(pw, pf, cout, 0, pb)
                    out["b%d/dw/w" % b] = np.ones((1, cin), np.float32)
                    out["b%d/dw/b" % b] = np.zeros(cin, np.float32)
                    out["b%d/dw/ksize" % b] = np.ones(cin, np.int32)
                    out["b%d/pw/w" % b] = np.ascontiguousarray(wf[:, 0, 0, :].T)
                    out["b%d/pw/b" % b] = (np.zeros(cout, np.float32) if pb is None else pb.data().reshape(-1).astype(np.float32))
                    modes.extend([MF.HYBRID_FLOAT, MF.HYBRID_FLOAT if codes is None else MF.HYBRID_ASYMMETRIC])
                    if codes is not None:
                        hy["hy/b%d/pw/w" % b] = np.ascontiguousarray(codes[:, 0, 0, :].T)
                        hy["hy/b%d/pw/scale" % b] = s
                pw_filters.append(cout)
                ksizes.append((1,))
                cur, cin = nxt, cout
                continue
            # depthwise groups: each reads the LAST k rows of its channel slice of the block's ring memory
            groups = []
            for dw in dws:
                f = self.t(dw.inputs[1])
                if len(f.shape) != 4 or f.shape[0] != 1 or f.shape[2] != 1:
                    self.fail(dw, "filter shape %s is not [1, k, 1, C]" % (f.shape,))
                if dw.opt(0, "b") != PADDING_VALID or dw.opt(2, "i", 1) != 1 or dw.opt(3, "i", 1) != 1 or dw.opt(6, "i", 1) != 1:
                    self.fail(dw, "depthwise conv must be VALID, stride 1, depth multiplier 1, no dilation (mixednet.py:195-197)")
                if dw.opt(4, "b") != ACT_NONE:
                    self.fail(dw, "depthwise conv with a fused activation")
                k, cg = f.shape[1], f.shape[3]
                x = self.t(dw.inputs[0])
                if x.shape != (1, k, 1, cg):
                    self.fail(dw, "input %s is not exactly one kernel window [1, %d, 1, %d] (StridedKeep, strided_drop.py:80-84)" % (x.shape, k, cg))
                src, keep = dw.inputs[0], None
                p = g.producer.get(src)
                if p is not None and p.code == OP_STRIDED_SLICE:
                    keep, src = p, p.inputs[0]
                    p = g.producer.get(src)
                slot = 0
                if p is not None and p.code in (OP_SPLIT_V, OP_SPLIT):
                    slot = p.outputs.index(src)
                    axis_t = self.t(p.inputs[2] if p.code == OP_SPLIT_V else p.inputs[0])
                    if int(axis_t.data().reshape(-1)[0]) not in (3, -1):
                        self.fail(p, "channel split along axis %d, expected the channel axis" % int(axis_t.data().reshape(-1)[0]))
                    mem = p.inputs[0] if p.code == OP_SPLIT_V else p.inputs[1]
                    split = p
                else:
                    mem, split = src, None
                rows = self.t(src).shape[1]
                if keep is not None:
                    # must keep the LAST k rows: begin row == rows - k
                    begin = self.t(keep.inputs[1]).data().reshape(-1)
                    if int(begin[1]) != rows - k and not (int(begin[1]) < 0 and int(begin[1]) == -k):
                        self.fail(keep, "StridedKeep begins at row %d, expected the last %d of %d rows" % (int(begin[1]), k, rows))
                elif rows != k:
                    self.fail(dw, "kernel %d on %d ring rows without a StridedKeep slice" % (k, rows))
                groups.append((slot, k, cg, dw, mem, split, f))
            groups.sort(key=lambda t: t[0])
            if [t[0] for t in groups] != list(range(len(groups))):
                self.fail(dws[0], "depthwise groups do not cover the SPLIT outputs 0..%d exactly once" % (len(groups) - 1))
            mems = {t[4] for t in groups}
            if len(mems) != 1 or (len(groups) > 1 and len({id(t[5]) for t in groups}) != 1):
                self.fail(dws[0], "depthwise groups of one block read different ring memories")
            mem = mems.pop()
            kmax = max(t[1] for t in groups)
            c_total = sum(t[2] for t in groups)
            if c_total != cin or self.t(mem).shape != (1, kmax, 1, cin):
                self.fail(dws[0], "block %d ring memory %s, expected [1, %d, 1, %d] (mixednet.py:193)" % (b, self.t(mem).shape, kmax, cin))
            ring, new = self.ring_memory(dws[0], mem, 1)
            if new != cur:
                self.fail(dws[0], "block %d does not read the previous layer's output" % b)
            want_split = [cin // len(groups)] * len(groups)
            want_split[0] += cin - sum(want_split)
            if [t[2] for t in groups] != want_split:
                self.fail(dws[0], "channel split %s differs from _split_channels %s (mixednet.py:132-136)" % ([t[2] for t in groups], want_split))
            # depthwise output: single group -> its output; several -> CONCATENATION along channels in group order
            if len(groups) == 1:
                d_out = groups[0][3].outputs[0]
            else:
                cons = g.consumers.get(groups[0][3].outputs[0], [])
                while len(cons) == 1 and cons[0].code == OP_STRIDED_SLICE:          # StridedDrop(0) if the converter kept it
                    cons = g.consumers.get(cons[0].outputs[0], [])
                if len(cons) != 1 or cons[0].code != OP_CONCATENATION or cons[0].opt(0, "i") not in (3, -1):
                    self.fail(groups[0][3], "depthwise group outputs are not concatenated along channels")
                cat = cons[0]
                srcs = [self.skip_back(x, (OP_STRIDED_SLICE,)) for x in cat.inputs]
                if srcs != [t[3].outputs[0] for t in groups]:
                    self.fail(cat, "channel concatenation order differs from the split order")
                d_out = cat.outputs[0]
            if self.t(d_out).shape != (1, 1, 1, cin):
                self.fail(dws[0], "depthwise output %s is not [1, 1, 1, %d]" % (self.t(d_out).shape, cin))
            # pointwise
            pf = self.t(pw.inputs[1])
            if len(pf.shape) != 4 or pf.shape[1:] != (1, 1, cin):
                self.fail(pw, "filter shape %s is not [filters, 1, 1, %d]" % (pf.shape, cin))
            if pw.inputs[0] != d_out:
                self.fail(pw, "1x1 conv does not read the block's depthwise output (residual connections are not supported)")
            if pw.opt(1, "i", 1) != 1 or pw.opt(2, "i", 1) != 1:
                self.fail(pw, "1x1 conv with a stride")
            relu, nxt = self.conv_act(pw, 3)
            if not relu:
                self.fail(pw, "1x1 conv without ReLU (mixednet.py:359)")
            cout = pf.shape[0]
            # container layout: depthwise taps [kmax, C], smaller kernels zero padded at the FRONT
            dw_w = np.zeros((kmax, cin), np.float64)
            dw_k = np.zeros(cin, np.int32)
            c_off = 0
            dw_bias_f, dw_bias_q, dw_scale = [], [], []
            hdw_w, hdw_s, dw_modes = np.zeros((kmax, cin), np.int8), np.zeros(cin, np.float32), []
            for slot, k, cg, dw, _, _, f in groups:
                bt = bias_of(dw, cg)
                if quantized:
                    dw_w[kmax - k:, c_off:c_off + cg] = f.data()[0, :, 0, :]
                else:
                    wf, codes, s = float_weights(dw, f, cg, 3, bt)
                    dw_w[kmax - k:, c_off:c_off + cg] = wf[0, :, 0, :]
                    dw_modes.append(MF.HYBRID_FLOAT if codes is None else MF.HYBRID_ASYMMETRIC)
                    if codes is not None:
                        hdw_w[kmax - k:, c_off:c_off + cg] = codes[0, :, 0, :]
                        hdw_s[c_off:c_off + cg] = s
                dw_k[c_off:c_off + cg] = k
                if quantized:
                    if f.dtype != np.int8 or np.any(f.zero_point != 0):
                        self.fail(dw, "depthwise weights must be symmetric int8")
                    s = f.scale.astype(np.float32)
                    dw_scale.append(np.repeat(s, cg) if s.size == 1 else s)
                    if dw_scale[-1].size != cg:
                        self.fail(dw, "%d weight scales for %d channels" % (s.size, cg))
                    dw_bias_q.append(np.zeros(cg, np.int32) if bt is None else bt.data().reshape(-1).astype(np.int32))
                    if self.t(dw.outputs[0]).per_tensor_q() != self.t(d_out).per_tensor_q():
                        self.fail(dw, "depthwise groups of one block have different output scales; the container holds one per block")
                else:
                    dw_bias_f.append(np.zeros(cg, np.float32) if bt is None else bt.data().reshape(-1).astype(np.float32))
                c_off += cg
            pw_w = pf.data()[:, 0, 0, :].T                                                # [cin, cout]
            pb = bias_of(pw, cout)
            act_q(self.t(d_out))
            act_q(self.t(nxt))
            if quantized:
                s_prev, s_d, s_p = scales[-3], scales[-2], scales[-1]
                sw = np.concatenate(dw_scale)
                ms = [quantize_multiplier(np.float64(s_prev) * np.float64(s) / np.float64(s_d)) for s in sw]
                out["q/b%d/dw/w" % b] = dw_w.astype(np.int8)
                out["q/b%d/dw/bias" % b] = np.concatenate(dw_bias_q)
                out["q/b%d/dw/mult" % b] = np.asarray([m for m, _ in ms], np.int32)
                out["q/b%d/dw/shift" % b] = np.asarray([s for _, s in ms], np.int32)
                weights_q("b%d/pw" % b, pf, pw_w, pb, cout, s_d, s_p)
            else:
                wf, codes, s = float_weights(pw, pf, cout, 0, pb)
                out["b%d/dw/w" % b] = dw_w.astype(np.float32)
                out["b%d/dw/b" % b] = np.concatenate(dw_bias_f)
                out["b%d/pw/w" % b] = np.ascontiguousarray(wf[:, 0, 0, :].T)
                out["b%d/pw/b" % b] = (np.zeros(cout, np.float32) if pb is None else pb.data().reshape(-1).astype(np.float32))
                modes.extend(dw_modes + [MF.HYBRID_FLOAT if codes is None else MF.HYBRID_ASYMMETRIC])
                if any(dw_modes):
                    hy["hy/b%d/dw/w" % b] = hdw_w
                    hy["hy/b%d/dw/scale" % b] = hdw_s
                if codes is not None:
                    hy["hy/b%d/pw/w" % b] = np.ascontiguousarray(codes[:, 0, 0, :].T)
                    hy["hy/b%d/pw/scale" % b] = s
            if not quantized:
                out["b%d/dw/ksize" % b] = dw_k
            pw_filters.append(cout)
            ksizes.append(tuple(t[1] for t in groups))
            cur, cin = nxt, cout

        # ---- head: Stream(Identity, ring T-1) -> Flatten -> Dense(1, sigmoid) (mixednet.py:362-384)
        fc, lg = compute[i], compute[i + 1]
        fw = self.t(fc.inputs[1])
        if len(fw.shape) != 2 or fw.shape[0] != 1 or fw.shape[1] % cin:
            self.fail(fc, "weights %s are not [1, T*%d]" % (fw.shape, cin))
        t_head = fw.shape[1] // cin
        if fc.opt(0, "b") != ACT_NONE:
            self.fail(fc, "dense head with a fused activation")
        memh = self.skip_back(fc.inputs[0])
        if t_head > 1:
            if self.t(memh).shape != (1, t_head, 1, cin):
                self.fail(fc, "flattened input %s is not the head ring [1, %d, 1, %d]" % (self.t(memh).shape, t_head, cin))
            ring, new = self.ring_memory(fc, memh, 1)
            if new != cur:
                self.fail(fc, "head does not read the last block's output")
        elif memh != cur:
            self.fail(fc, "head does not read the last block's output")
        if lg.inputs[0] != fc.outputs[0]:
            self.fail(lg, "LOGISTIC does not read the dense output")
        fb = bias_of(fc, 1)
        hw = fw.data().reshape(t_head, cin)
        act_q(self.t(fc.outputs[0]))
        act_q(self.t(lg.outputs[0]))
        final = lg.outputs[0]
        cons = g.consumers.get(final, [])
        if quantized:
            if len(cons) != 1 or cons[0].code != OP_QUANTIZE or cons[0].outputs[0] != g.outputs[0] or tout.dtype != np.uint8:
                self.fail(lg, "int8 graph must end in QUANTIZE to uint8 (utils.py:338)")
            so, zo = tout.per_tensor_q()
            if scales[-1] != np.float32(1.0 / 256.0) or zps[-1] != -128 or so != np.float32(1.0 / 256.0) or zo != 0:
                self.fail(lg, "LOGISTIC output must be scale 1/256, zero point -128 (uint8: 0); got %r / %r and %r / %r" % (scales[-1], zps[-1], so, zo))
            weights_q("head", fw, hw, fb, 1, scales[-3], scales[-2])
            out["q/logistic_lut"] = logistic_lut(scales[-2], zps[-2], zps[-1])
            out["q/scales"] = np.asarray(scales, np.float32)
            out["q/zps"] = np.asarray(zps, np.int32)
        else:
            if final != g.outputs[0] or tout.dtype != np.float32:
                self.fail(lg, "float graph must end in LOGISTIC")
            wf, codes, s = float_weights(fc, fw, 1, 0, fb)
            out["head/w"] = np.ascontiguousarray(wf.reshape(t_head, cin))
            out["head/b"] = np.zeros(1, np.float32) if fb is None else fb.data().reshape(-1).astype(np.float32)
            # FullyConnectedOptions.asymmetric_quantize_inputs (field 3) picks the hybrid kernel's input quantiser
            modes.append(MF.HYBRID_FLOAT if codes is None else
                         (MF.HYBRID_ASYMMETRIC if fc.opt(3, "B") else MF.HYBRID_SYMMETRIC))
            if codes is not None:
                hy["hy/head/w"] = np.ascontiguousarray(codes.reshape(t_head, cin))
                hy["hy/head/scale"] = s

        self.check_initial_state(zps if quantized else None)
        arch = MF.Arch(f0, k0, stride, tuple(pw_filters), tuple(ksizes), t_head)
        out["arch"] = arch.encode()
        if any(modes):
            assert len(modes) == len(MF.hybrid_slots(arch))
            out["hy/mode"] = np.asarray(modes, np.int32)
            out.update(hy)
        return out

    def check_initial_state(self, zps):
        """The engine starts every ring at real zero (mww_reset); a CALL_ONCE initialiser that says otherwise is refused."""
        if len(self.g.subgraphs) < 2:
            return
        tensors, ops, _, _ = self.g.subgraphs[1]
        for op in ops:
            if op.code != OP_ASSIGN_VARIABLE:
                continue
            v = tensors[op.inputs[1]]
            if not v.is_constant:
                continue
            d = v.data()
            want = int(v.zero_point[0]) if (v.dtype == np.int8 and v.zero_point.size) else 0
            if np.any(d != want):
                raise TfliteError("variable initialiser %r is not all (real) zero; the streaming engine resets rings to zero" % v.name)


def tensors_from_tflite(blob: bytes) -> dict:
    """TFL3 flatbuffer bytes -> the tensor dictionary ``model_file.write_container`` serialises.
    Whatever is wrong with the bytes -- truncated file, offsets pointing outside it, indices outside a vector, shapes that do
    not multiply out -- surfaces as TfliteError: a file this reader cannot vouch for is rejected, never half-read."""
    blob = bytes(blob)
    if len(blob) < 8 or blob[4:8] != FILE_IDENTIFIER:
        raise TfliteError("not a TFL3 flatbuffer (file identifier missing)")
    try:
        return _Recogniser(Graph(blob)).run()
    except TfliteError:
        raise
    except (struct.error, IndexError, KeyError, ValueError, OverflowError, TypeError, AttributeError, RecursionError, MemoryError, ZeroDivisionError) as exc:
        raise TfliteError("malformed flatbuffer (%s: %s)" % (type(exc).__name__, exc)) from exc


def is_tflite(blob: bytes) -> bool:
    return len(blob) >= 8 and bytes(blob[4:8]) == FILE_IDENTIFIER


def container_from_tflite(blob: bytes) -> bytes:
    return MF.write_container(tensors_from_tflite(blob))
