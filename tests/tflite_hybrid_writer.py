"""Test infrastructure: the float streaming MixedNet of ``tests/tflite_writer.py`` with the weight tensors that dynamic-range
quantisation stores as int8 (``utils.convert_saved_model_to_tflite`` without a representative dataset, utils.py:328): each
chosen CONV_2D / DEPTHWISE_CONV_2D / FULLY_CONNECTED weight becomes symmetric int8 with one float32 scale per output channel
(scale = max|w| / 127, zero points 0), and a hybrid dense head carries FullyConnectedOptions.asymmetric_quantize_inputs
(field 3).  Activations, biases and ring variables stay float32.

Built on ``tflite_writer.write_streaming_mixednet``: a GraphWriter subclass rewrites the chosen weight tensors just before
serialisation.  Not TensorFlow output (see tflite_writer.py)."""

from __future__ import annotations

import contextlib
import re

import numpy as np

import tflite_writer as TW

# weight tensor names of tflite_writer -> (model_file.hybrid_slots name, output-channel dimension)
_WEIGHTS = [
    (re.compile(r"^stream/conv2d/kernel$"), lambda m: "first_conv", 0),
    (re.compile(r"^dw_(\d+)_(\d+)/kernel$"), lambda m: "b%s/dw%s" % (m.group(1), m.group(2)), 3),
    (re.compile(r"^pw_(\d+)/kernel$"), lambda m: "b%s/pw" % m.group(1), 0),
    (re.compile(r"^dense/kernel$"), lambda m: "head", 0),
]


def quantize_weights(w: np.ndarray, qdim: int):
    """symmetric per-channel int8 along qdim -> (codes, float32 scales)"""
    mx = np.abs(w).max(axis=tuple(i for i in range(w.ndim) if i != qdim)).astype(np.float32)
    s = np.where(mx > 0, mx / np.float32(127.0), np.float32(1.0)).astype(np.float32)
    shape = [1] * w.ndim
    shape[qdim] = -1
    return np.clip(np.round(w / s.reshape(shape)), -127, 127).astype(np.int8), s


@contextlib.contextmanager
def _writer(hybrid, fc_asymmetric, edit):
    base = TW.GraphWriter

    class HybridGraphWriter(base):
        def serialise(self, *a, **kw):
            fc_hybrid = False
            for t in self.tensors:
                for pat, slot, qdim in _WEIGHTS:
                    m = pat.match(t["name"])
                    if m is None or t["type"] != TW.T_FLOAT32 or not t["buffer"]:
                        continue
                    w = np.frombuffer(self.buffers[t["buffer"]], np.float32).reshape(t["shape"])
                    if not hybrid(slot(m), w.size):
                        continue
                    codes, s = quantize_weights(w, qdim)
                    self.buffers[t["buffer"]] = codes.tobytes()
                    t.update(type=TW.T_INT8, scale=s, zero_point=np.zeros(s.size, np.int64), qdim=qdim)
                    fc_hybrid |= slot(m) == "head"
            if fc_hybrid and fc_asymmetric:
                for name, _, _, o in self.ops:
                    if name == "FULLY_CONNECTED":
                        o["asymmetric_quantize_inputs"] = True
            if edit is not None:
                edit({t["name"]: t for t in self.tensors}, self)
            return super().serialise(*a, **kw)

        def _options(self, b, name, o):
            if name == "FULLY_CONNECTED" and o.get("asymmetric_quantize_inputs"):
                b.start()
                b.scalar(0, "b", 0)
                b.scalar(3, "B", 1)
                return b.end()
            return super()._options(b, name, o)

    TW.GraphWriter = HybridGraphWriter
    try:
        yield
    finally:
        TW.GraphWriter = base


def write_hybrid_mixednet(tensors: dict, hybrid, fc_asymmetric: bool = True, edit=None, shuffle_seed=None) -> bytes:
    """fp32 ``model_file`` tensors -> TFL3 bytes of the float streaming graph with int8 weights where
    ``hybrid(op, n_elements)`` says so (``op`` a ``model_file.hybrid_slots`` name).  Converter-like: ``n_elements >= 1024``.
    edit(tensors_by_name, graph_writer): optional change to the graph just before serialisation (refusal tests)."""
    with _writer(hybrid, fc_asymmetric, edit):
        return TW.write_streaming_mixednet(tensors, shuffle_seed=shuffle_seed)
