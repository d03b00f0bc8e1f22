"""oracle/mixednet_ref.py -- CPU ORACLE (test infrastructure, NOT product code).

NumPy restatement of the reference's streaming MixedNet, one model step at a time, written
literally after the Keras graph so that every ring-buffer concat / slice is visible:

  * topology ............ microwakeword/mixednet.py:278-386 (model), :168-231 (MixConv),
                          :132-136 (_split_channels)
  * ring semantics ...... microwakeword/layers/stream.py:581-595 (concat(state, input),
                          state <- last N rows, cell(memory)); ring sizes :241-255
  * StridedKeep ......... microwakeword/layers/strided_drop.py:80-84 (last k rows when streaming)
  * streaming input ..... microwakeword/layers/modes.py:57-64 -> (stride, 40), batch 1 (utils.py:218-222)
  * driver loop ......... microwakeword/inference.py:98-123 (chunking + per-chunk invoke)
  * int8 contract ....... microwakeword/utils.py:289-348 (int8 in, uint8 out, quantised state
                          variables, representative range pinned to [0, 26]) executed with the
                          published TFLite int8 kernel semantics (SURVEY.md Appendix C):
                          per-channel symmetric weights, SaturatingRoundingDoublingHighMul +
                          RoundingDivideByPOT requantisation, LUT logistic.

      *** PARITY UNPINNED ***
The reference runs this graph inside tf.lite.Interpreter / Keras, neither of which exists in
this image, and it ships no golden vectors (SURVEY.md 8c).  This file is therefore the
definition every GPU parity test is measured against.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this module.
"""

from __future__ import annotations

import numpy as np

NUM_FEATURES = 40
FEATURE_SCALE = np.float32(0.0390625)
BN_EPS = 1e-3  # tf.keras.layers.BatchNormalization default epsilon


# --------------------------------------------------------------------------------------
# architecture helpers (duplicated on purpose: the oracle does not import the product)

class Spec:
    def __init__(self, first_conv_filters=32, first_conv_kernel_size=5, stride=3,
                 pointwise_filters=(64, 64, 64, 64),
                 mixconv_kernel_sizes=((5,), (7, 11), (9, 15), (23,)), head_rows=17):
        self.first_conv_filters = first_conv_filters
        self.first_conv_kernel_size = first_conv_kernel_size
        self.stride = stride
        self.pointwise_filters = tuple(pointwise_filters)
        self.mixconv_kernel_sizes = tuple(tuple(k) for k in mixconv_kernel_sizes)
        self.head_rows = head_rows

    @property
    def n_blocks(self):
        return len(self.pointwise_filters)

    def cin(self, i):
        return self.first_conv_filters if i == 0 else self.pointwise_filters[i - 1]

    def splits(self, i):
        # mixednet.py:132-136
        total, groups = self.cin(i), len(self.mixconv_kernel_sizes[i])
        split = [total // groups for _ in range(groups)]
        split[0] += total - sum(split)
        return split

    def encode(self):
        v = [self.first_conv_filters, self.first_conv_kernel_size, self.stride, NUM_FEATURES,
             self.n_blocks, self.head_rows]
        for f, ks in zip(self.pointwise_filters, self.mixconv_kernel_sizes):
            v += [f, len(ks)] + list(ks) + [0] * (4 - len(ks))
        return np.asarray(v, np.int32)

    @staticmethod
    def decode(v):
        v = [int(x) for x in v]
        pw, ks = [], []
        for b in range(v[4]):
            o = 6 + 6 * b
            pw.append(v[o])
            ks.append(tuple(v[o + 2:o + 2 + v[o + 1]]))
        return Spec(v[0], v[1], v[2], pw, ks, v[5])


OKAY_NABU = Spec()


# --------------------------------------------------------------------------------------
# synthetic Keras-form parameters (no trained weights exist in this environment)

def init_synthetic(spec: Spec = OKAY_NABU, seed: int = 0) -> dict:
    """Deterministic, well-conditioned Keras-form parameters (SURVEY.md section 7 step 2).

    He-normal kernels, BN gamma in [0.5, 1.5], small BN beta / moving mean, moving variance
    near the layer's actual output variance, and a dense layer scaled so that the
    probabilities over typical features cover most of (0, 1).
    """
    rng = np.random.default_rng(seed)
    p = {}
    k0, f0 = spec.first_conv_kernel_size, spec.first_conv_filters
    # features live in [0, 26]; scale the first kernel so activations stay O(1)
    p["first_conv/kernel"] = (rng.normal(0, 1, (k0, NUM_FEATURES, f0)) * np.sqrt(2.0 / (k0 * NUM_FEATURES)) / 6.0).astype(np.float32)
    for i in range(spec.n_blocks):
        cin, cout = spec.cin(i), spec.pointwise_filters[i]
        dws, dbs = [], []
        if max(spec.mixconv_kernel_sizes[i]) > 1:          # mixednet.py:346-348: a block whose largest kernel is 1 has NO MixConv layer
            for n, k in zip(spec.splits(i), spec.mixconv_kernel_sizes[i]):
                dws.append((rng.normal(0, 1, (k, n)) * np.sqrt(2.0 / k)).astype(np.float32))
                dbs.append(rng.normal(0, 0.05, n).astype(np.float32))
        p["b%d/dw/kernels" % i] = dws
        p["b%d/dw/biases" % i] = dbs
        p["b%d/pw/kernel" % i] = (rng.normal(0, 1, (cin, cout)) * np.sqrt(2.0 / cin)).astype(np.float32)
        p["b%d/bn/gamma" % i] = rng.uniform(0.5, 1.5, cout).astype(np.float32)
        p["b%d/bn/beta" % i] = rng.normal(0, 0.2, cout).astype(np.float32)
        p["b%d/bn/mean" % i] = rng.normal(0, 0.3, cout).astype(np.float32)
        p["b%d/bn/var" % i] = rng.uniform(1.5, 3.0, cout).astype(np.float32)
    n_flat = spec.head_rows * spec.pointwise_filters[-1]
    p["dense/kernel"] = (rng.normal(0, 1, (n_flat, 1)) * (2.5 / np.sqrt(n_flat))).astype(np.float32)
    p["dense/bias"] = np.asarray([-0.3], np.float32)
    return p


def fold_bn(spec: Spec, p: dict) -> dict:
    """Keras-form -> inference-form tensors with BatchNorm folded into the 1x1 conv, named as the
    product's model container names them (microwakeword_b200/model_file.py)."""
    t = {"arch": spec.encode(), "first_conv/w": p["first_conv/kernel"].astype(np.float32)}
    for i in range(spec.n_blocks):
        ks = spec.mixconv_kernel_sizes[i]
        kmax, cin = max(ks), spec.cin(i)
        w = np.zeros((kmax, cin), np.float32)
        b = np.zeros(cin, np.float32)
        kk = np.zeros(cin, np.int32)
        c0 = 0
        if kmax == 1:
            # no MixConv in the graph (mixednet.py:346-348): the container's depthwise stage is the exact identity
            # (tap 1, bias 0), so every kernel keeps one uniform block structure
            w[:] = 1.0
            kk[:] = 1
        for kern, bias, k in zip(p["b%d/dw/kernels" % i], p["b%d/dw/biases" % i], ks if kmax > 1 else ()):
            n = kern.shape[1]
            w[kmax - k:, c0:c0 + n] = kern  # the LAST k rows of the ring window are used
            b[c0:c0 + n] = bias
            kk[c0:c0 + n] = k
            c0 += n
        t["b%d/dw/w" % i], t["b%d/dw/b" % i], t["b%d/dw/ksize" % i] = w, b, kk
        g = (p["b%d/bn/gamma" % i].astype(np.float64) / np.sqrt(p["b%d/bn/var" % i].astype(np.float64) + BN_EPS))
        t["b%d/pw/w" % i] = (p["b%d/pw/kernel" % i].astype(np.float64) * g[None, :]).astype(np.float32)
        t["b%d/pw/b" % i] = (p["b%d/bn/beta" % i].astype(np.float64) - p["b%d/bn/mean" % i].astype(np.float64) * g).astype(np.float32)
    t["head/w"] = p["dense/kernel"].reshape(spec.head_rows, spec.pointwise_filters[-1]).astype(np.float32)
    t["head/b"] = p["dense/bias"].astype(np.float32)
    return t


def _sigmoid(x):
    x = np.float32(x)
    return np.float32(1.0) / (np.float32(1.0) + np.exp(-x, dtype=np.float32))


# --------------------------------------------------------------------------------------
# fp32 streaming model, Keras semantics (BN applied explicitly, not folded)

class KerasStreamingF32:
    """One Stream()/MixConv()/Conv2D/BN/ReLU layer per line of mixednet.py:307-386, batch 1."""

    def __init__(self, spec: Spec, params: dict):
        self.spec, self.p = spec, params
        self.reset()

    def reset(self):
        s = self.spec
        # stream.py:420-425 zeros initializer
        self.st_first = np.zeros((s.first_conv_kernel_size - 1 - (s.stride - 1), NUM_FEATURES), np.float32)
        self.st_block = [np.zeros((max(s.mixconv_kernel_sizes[i]) - 1, s.cin(i)), np.float32) for i in range(s.n_blocks)]
        self.st_head = np.zeros((s.head_rows - 1, s.pointwise_filters[-1]), np.float32)

    def step(self, x: np.ndarray) -> np.float32:
        """x: float32 [stride, 40] -> probability (inference.py:113-119 one invoke)."""
        s, p = self.spec, self.p
        x = np.asarray(x, np.float32).reshape(s.stride, NUM_FEATURES)
        # Stream(Conv2D(k,1) stride (s,1), valid, no bias): stream.py:581-593
        mem = np.concatenate([self.st_first, x], 0)
        self.st_first = mem[-self.st_first.shape[0]:] if self.st_first.shape[0] else self.st_first
        net = np.einsum("kf,kfo->o", mem, p["first_conv/kernel"], dtype=np.float32)[None, :]
        net = np.maximum(net, np.float32(0))
        for i in range(s.n_blocks):
            ks = s.mixconv_kernel_sizes[i]
            if max(ks) > 1:                   # mixednet.py:346-348: no MixConv at all when the largest kernel is 1
                # MixConv: Stream(Identity, ring=max(k)-1)  mixednet.py:202-206
                mem = np.concatenate([self.st_block[i], net], 0)
                if self.st_block[i].shape[0]:
                    self.st_block[i] = mem[-self.st_block[i].shape[0]:]
                outs, c0 = [], 0
                for kern, bias, k, n in zip(p["b%d/dw/kernels" % i], p["b%d/dw/biases" % i], ks, s.splits(i)):
                    part = mem[:, c0:c0 + n]
                    if len(ks) > 1:
                        part = part[-k:]          # StridedKeep, strided_drop.py:80-84
                    outs.append((part * kern).sum(0, dtype=np.float32) + bias)  # DepthwiseConv2D valid
                    c0 += n
                net = np.concatenate(outs)[None, :].astype(np.float32)
            # Conv2D 1x1 no bias -> BatchNormalization (inference form) -> ReLU   mixednet.py:349-360
            net = (net @ p["b%d/pw/kernel" % i]).astype(np.float32)
            inv = (p["b%d/bn/gamma" % i] / np.sqrt(p["b%d/bn/var" % i] + np.float32(BN_EPS))).astype(np.float32)
            net = (net - p["b%d/bn/mean" % i]) * inv + p["b%d/bn/beta" % i]
            net = np.maximum(net, np.float32(0)).astype(np.float32)
        # Stream(Identity, ring=T-1) -> Flatten -> Dense(1, sigmoid)   mixednet.py:362-384
        mem = np.concatenate([self.st_head, net], 0)
        if self.st_head.shape[0]:                    # a 1-row head keeps no history: mem[-0:] would be the whole window
            self.st_head = mem[-self.st_head.shape[0]:]
        logit = (mem.reshape(1, -1) @ p["dense/kernel"])[0, 0] + p["dense/bias"][0]
        return _sigmoid(logit)


# --------------------------------------------------------------------------------------
# fp32 streaming model, inference form (BN folded) -- what the product's fp32 path is graded on

class FoldedStreamingF32:
    def __init__(self, tensors: dict):
        self.t = tensors
        self.spec = Spec.decode(tensors["arch"])
        self.reset()

    def reset(self):
        s = self.spec
        self.st_first = np.zeros((s.first_conv_kernel_size - 1 - (s.stride - 1), NUM_FEATURES), np.float32)
        self.st_block = [np.zeros((max(s.mixconv_kernel_sizes[i]) - 1, s.cin(i)), np.float32) for i in range(s.n_blocks)]
        self.st_head = np.zeros((s.head_rows - 1, s.pointwise_filters[-1]), np.float32)

    def step(self, x, want_logit=False):
        s, t = self.spec, self.t
        x = np.asarray(x, np.float32).reshape(s.stride, NUM_FEATURES)
        mem = np.concatenate([self.st_first, x], 0)
        if self.st_first.shape[0]:
            self.st_first = mem[-self.st_first.shape[0]:]
        net = np.maximum(np.einsum("kf,kfo->o", mem, t["first_conv/w"], dtype=np.float32), np.float32(0))
        for i in range(s.n_blocks):
            mem = np.concatenate([self.st_block[i], net[None, :]], 0)
            if self.st_block[i].shape[0]:            # a 0-row ring (1-tap block) stays empty: mem[-0:] would be the whole window
                self.st_block[i] = mem[-self.st_block[i].shape[0]:]
            d = (mem * t["b%d/dw/w" % i]).sum(0, dtype=np.float32) + t["b%d/dw/b" % i]
            net = np.maximum((d @ t["b%d/pw/w" % i]).astype(np.float32) + t["b%d/pw/b" % i], np.float32(0))
        mem = np.concatenate([self.st_head, net[None, :]], 0)
        if self.st_head.shape[0]:                    # a 1-row head keeps no history: mem[-0:] would be the whole window
            self.st_head = mem[-self.st_head.shape[0]:]
        logit = np.float32((mem * t["head/w"]).sum(dtype=np.float32) + t["head/b"][0])
        return logit if want_logit else _sigmoid(logit)

    def activations(self, x):
        """Like step() but returns every intermediate tensor (used for int8 calibration)."""
        s, t = self.spec, self.t
        acts = {}
        x = np.asarray(x, np.float32).reshape(s.stride, NUM_FEATURES)
        acts["in"] = x
        mem = np.concatenate([self.st_first, x], 0)
        if self.st_first.shape[0]:
            self.st_first = mem[-self.st_first.shape[0]:]
        net = np.maximum(np.einsum("kf,kfo->o", mem, t["first_conv/w"], dtype=np.float32), np.float32(0))
        acts["c0"] = net
        for i in range(s.n_blocks):
            mem = np.concatenate([self.st_block[i], net[None, :]], 0)
            if self.st_block[i].shape[0]:            # a 0-row ring (1-tap block) stays empty: mem[-0:] would be the whole window
                self.st_block[i] = mem[-self.st_block[i].shape[0]:]
            d = (mem * t["b%d/dw/w" % i]).sum(0, dtype=np.float32) + t["b%d/dw/b" % i]
            acts["d%d" % (i + 1)] = d
            net = np.maximum((d @ t["b%d/pw/w" % i]).astype(np.float32) + t["b%d/pw/b" % i], np.float32(0))
            acts["p%d" % (i + 1)] = net
        mem = np.concatenate([self.st_head, net[None, :]], 0)
        if self.st_head.shape[0]:                    # a 1-row head keeps no history: mem[-0:] would be the whole window
            self.st_head = mem[-self.st_head.shape[0]:]
        acts["fc"] = np.float32((mem * t["head/w"]).sum(dtype=np.float32) + t["head/b"][0])
        return acts


# --------------------------------------------------------------------------------------
# float64 streaming model with a running bound on the error of ANY fp32 evaluation of the same folded graph

U32 = 2.0 ** -24            # unit roundoff of float32
PROB_SLACK = 2.0 ** -20     # expf and the division of a float32 sigmoid


def gamma(n: int) -> float:
    """gamma_n = n u / (1 - n u): a sum of n products in float32, in any order, with or without fused multiply-adds, is
    within gamma_n * sum |products| of the exact sum (Higham, Accuracy and Stability of Numerical Algorithms, 3.1)."""
    return n * U32 / (1.0 - n * U32)


def _dot_bound(x, ex, w, b=None, axis=0):
    """exact (float64) value of sum(x * w, axis) (+ b) and the bound on its fp32 evaluation from inputs known to within ex:
    E = sum |w| ex + gamma_{n+1} (sum |w| (|x| + ex) + |b|)  -- the n + 1 counts the bias add; |x| + ex bounds the
    fp32 input the evaluation actually multiplies."""
    aw = np.abs(w)
    n = x.shape[axis] + (b is not None)
    y = (x * w).sum(axis)
    e = (ex * aw).sum(axis) + gamma(n) * ((np.abs(x) + ex) * aw).sum(axis)
    if b is not None:
        y = y + b
        e = e + gamma(n) * np.abs(b)
    return y, e


def _relu_bound(y, e):
    """ReLU of a value known to within e: relu is 1-Lipschitz, and an input below -e is negative in fp32 too, so its output
    is exactly 0 there -- the bound is the widest move of relu over [y - e, y + e]"""
    r = np.maximum(y, 0.0)
    return r, np.maximum(np.maximum(y + e, 0.0) - r, r - np.maximum(y - e, 0.0))


class StreamingF64:
    """FoldedStreamingF32's graph in float64.  Next to every value it carries E, a bound on how far an fp32 evaluation of
    the same graph (any summation order, fmaf or not) can be from it: inputs are exact (E = 0; a uint16 feature x
    0.0390625 is exact in float32), every dot product adds its rounding bound (_dot_bound), ReLU passes E through (_relu_bound), every
    ring entry keeps its own E, and |p - p64| <= E_logit / 4 + PROB_SLACK (the sigmoid's slope is at most 1/4).
    The bound assumes nothing about loop structure, so it checks a kernel whatever order it sums in."""

    def __init__(self, tensors: dict):
        self.spec = Spec.decode(tensors["arch"])
        self.w0 = tensors["first_conv/w"].astype(np.float64).reshape(-1, self.spec.first_conv_filters)
        self.blk = [tuple(tensors["b%d/%s" % (i, n)].astype(np.float64) for n in ("dw/w", "dw/b", "pw/w", "pw/b"))
                    for i in range(self.spec.n_blocks)]
        self.head_w = tensors["head/w"].astype(np.float64)
        self.head_b = float(tensors["head/b"][0])
        self.reset()

    def reset(self):
        s = self.spec
        self.st_first = np.zeros((s.first_conv_kernel_size - s.stride, NUM_FEATURES))
        self.st_block = [np.zeros((max(s.mixconv_kernel_sizes[i]) - 1, s.cin(i))) for i in range(s.n_blocks)]
        self.st_head = np.zeros((s.head_rows - 1, s.pointwise_filters[-1]))
        self.e_block = [np.zeros_like(r) for r in self.st_block]
        self.e_head = np.zeros_like(self.st_head)

    @staticmethod
    def _push(ring, row):
        mem = np.concatenate([ring, row[None, :]], 0)
        return mem, (mem[1:] if ring.shape[0] else ring)

    def step(self, x):
        """x: [stride, 40] rows as the fp32 model sees them -> (p64, bound on |p - p64|, logit64, bound on the logit)"""
        s = self.spec
        x = np.asarray(x, np.float32).astype(np.float64).reshape(s.stride, NUM_FEATURES)
        mem = np.concatenate([self.st_first, x], 0)
        if self.st_first.shape[0]:
            self.st_first = mem[-self.st_first.shape[0]:]
        flat = mem.reshape(-1, 1)
        net, e = _relu_bound(*_dot_bound(flat, np.zeros_like(flat), self.w0))
        for i, (dw, db, pw, pb) in enumerate(self.blk):
            mem, self.st_block[i] = self._push(self.st_block[i], net)
            emem, self.e_block[i] = self._push(self.e_block[i], e)
            d, ed = _dot_bound(mem, emem, dw, db)
            net, e = _relu_bound(*_dot_bound(d[:, None], ed[:, None], pw, pb))
        mem, self.st_head = self._push(self.st_head, net)
        emem, self.e_head = self._push(self.e_head, e)
        logit, el = _dot_bound(mem.reshape(-1), emem.reshape(-1), self.head_w.reshape(-1), np.float64(self.head_b))
        p = 1.0 / (1.0 + np.exp(-logit))
        return float(p), float(el / 4.0 + PROB_SLACK), float(logit), float(el)

    def state(self):
        """(values, bounds) of the ring state in the engine's per-stream layout: first-conv ring, block rings, head ring"""
        vals = np.concatenate([self.st_first.ravel()] + [r.ravel() for r in self.st_block] + [self.st_head.ravel()])
        errs = np.concatenate([np.zeros(self.st_first.size)] + [r.ravel() for r in self.e_block] + [self.e_head.ravel()])
        return vals, errs


def nonstreaming_logits(tensors: dict, spectrogram: np.ndarray) -> np.ndarray:
    """Whole-clip (NON_STREAM_INFERENCE) forward with 'valid' convs (README.md:27-28): returns the
    logit for every position where the non-streaming graph has a full receptive field."""
    s = Spec.decode(tensors["arch"])
    x = np.asarray(spectrogram, np.float32)
    k0 = s.first_conv_kernel_size
    n0 = (x.shape[0] - k0) // s.stride + 1
    net = np.stack([np.einsum("kf,kfo->o", x[j * s.stride:j * s.stride + k0], tensors["first_conv/w"], dtype=np.float32) for j in range(n0)])
    net = np.maximum(net, 0)
    for i in range(s.n_blocks):
        w, b = tensors["b%d/dw/w" % i], tensors["b%d/dw/b" % i]
        kmax = w.shape[0]
        n = net.shape[0] - kmax + 1
        d = np.stack([(net[j:j + kmax] * w).sum(0, dtype=np.float32) + b for j in range(n)])
        net = np.maximum(d @ tensors["b%d/pw/w" % i] + tensors["b%d/pw/b" % i], 0).astype(np.float32)
    n = net.shape[0] - s.head_rows + 1
    return np.asarray([(net[j:j + s.head_rows] * tensors["head/w"]).sum(dtype=np.float32) + tensors["head/b"][0] for j in range(n)], np.float32)


# --------------------------------------------------------------------------------------
# reference driver loop (inference.py:82-125)

def predict_spectrogram(model, spectrogram: np.ndarray, stride=None, quantized=False, in_scale=None, in_zp=None):
    """Restates Model.predict_spectrogram: dtype normalisation (:93-96), chunking (:98-105),
    per-chunk invoke (:109-123).  `model` is any object with .spec and .step()."""
    spec = model.spec
    slices = spec.stride
    stride = slices if stride is None else stride
    if np.issubdtype(spectrogram.dtype, np.uint16):
        spectrogram = spectrogram.astype(np.float32) * FEATURE_SCALE
    elif np.issubdtype(spectrogram.dtype, np.float64):
        spectrogram = spectrogram.astype(np.float32)
    out = []
    for last in range(slices, len(spectrogram) + 1, stride):
        chunk = spectrogram[last - slices:last]
        if len(chunk) != slices:
            continue
        if quantized and spectrogram.dtype != np.int8:
            chunk = quantize_input(chunk, in_scale, in_zp)       # inference.py:127-147
        y = model.step(chunk)
        if quantized:
            y = np.float32(1 / 255.0 * (np.float32(y) - 0))       # inference.py:162-170 (zp 0 for uint8 out)
        out.append(y)
    return out


def quantize_input(data: np.ndarray, scale, zp) -> np.ndarray:
    """inference.py:127-147 -- float divide, add zero point, astype(int8): truncation toward zero
    and C-style wrap, no clamp."""
    v = np.asarray(data, np.float32) / np.float32(scale) + np.float32(zp)
    return v.astype(np.int32).astype(np.int8)  # numpy float->int8 direct cast is UB out of range; wrap explicitly


# --------------------------------------------------------------------------------------
# TFLite int8 arithmetic (SURVEY.md Appendix C)

def quantize_multiplier(real: float):
    """TFLite QuantizeMultiplier: real = M0 * 2^(shift-31), M0 in [2^30, 2^31)."""
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


def srdhm(a, b):
    """SaturatingRoundingDoublingHighMul on int64 numpy arrays holding int32 values."""
    a = np.asarray(a, np.int64)
    b = np.asarray(b, np.int64)
    ab = a * b
    nudge = np.where(ab >= 0, 1 << 30, 1 - (1 << 30))
    t = ab + nudge
    # C++ integer division truncates toward zero
    q = np.where(t >= 0, t >> 31, -((-t) >> 31))
    overflow = (a == -(1 << 31)) & (b == -(1 << 31))
    return np.where(overflow, (1 << 31) - 1, q)


def rounding_divide_by_pot(x, exponent):
    x = np.asarray(x, np.int64)
    exponent = np.asarray(exponent, np.int64)
    mask = (np.int64(1) << exponent) - 1
    rem = x & mask
    thr = (mask >> 1) + (x < 0)
    return (x >> exponent) + (rem > thr)


def mbqm(x, mult, shift):
    """MultiplyByQuantizedMultiplier (double-rounding variant, the TFLite default)."""
    shift = np.asarray(shift, np.int64)
    left = np.maximum(shift, 0)
    right = np.maximum(-shift, 0)
    return rounding_divide_by_pot(srdhm(np.asarray(x, np.int64) * (np.int64(1) << left), mult), right)


def _act_qparams(lo, hi):
    """Asymmetric int8 params for a [lo, hi] float range that is forced to contain 0."""
    lo, hi = min(float(lo), 0.0), max(float(hi), 0.0)
    if hi == lo:
        return np.float32(1.0), 0
    scale = (hi - lo) / 255.0
    zp = int(np.round(-128 - lo / scale))
    return np.float32(scale), int(np.clip(zp, -128, 127))


def quantize_model(tensors: dict, calib_features: np.ndarray) -> dict:
    """Post-training int8 quantisation of the folded fp32 graph, following the contract of
    utils.py:289-348: per-tensor asymmetric int8 activations calibrated on a representative
    set whose input range is pinned to [0, 26] (:308-313), per-output-channel symmetric int8
    conv weights, int32 biases at scale s_in * s_w, quantised state variables (:333) sharing
    the params of the tensor they buffer, int8 input, uint8 output (:337-338).

    calib_features: float32 [N, stride, 40] chunks fed sequentially through the fp32 model.
    """
    spec = Spec.decode(tensors["arch"])
    f32 = FoldedStreamingF32(tensors)
    lo, hi = {}, {}
    for chunk in calib_features:
        for name, a in f32.activations(chunk).items():
            lo[name] = min(lo.get(name, np.inf), float(np.min(a)))
            hi[name] = max(hi.get(name, -np.inf), float(np.max(a)))
    lo["in"], hi["in"] = 0.0, 26.0  # utils.py:308-313
    names = ["in", "c0"] + [n for i in range(spec.n_blocks) for n in ("d%d" % (i + 1), "p%d" % (i + 1))] + ["fc", "prob"]
    scales, zps = {}, {}
    for n in names[:-1]:
        scales[n], zps[n] = _act_qparams(lo[n], hi[n])
    identity = [max(ks) == 1 for ks in spec.mixconv_kernel_sizes]
    for i, ident in enumerate(identity):
        if ident:   # no MixConv, hence no tensor between the previous activation and the 1x1 conv (mixednet.py:346-348)
            prev = "c0" if i == 0 else "p%d" % i
            scales["d%d" % (i + 1)], zps["d%d" % (i + 1)] = scales[prev], zps[prev]
    scales["prob"], zps["prob"] = np.float32(1.0 / 256.0), -128  # TFLite LOGISTIC int8 output params

    q = {"arch": tensors["arch"].copy()}
    q["q/scales"] = np.asarray([scales[n] for n in names], np.float32)
    q["q/zps"] = np.asarray([zps[n] for n in names], np.int32)

    def conv_layer(prefix, w, bias, s_in, s_out, axis_out):
        # per-output-channel symmetric weights
        wmax = np.abs(w).max(axis=tuple(a for a in range(w.ndim) if a != axis_out))
        s_w = np.where(wmax > 0, wmax / 127.0, 1.0).astype(np.float64)
        shape = [1] * w.ndim
        shape[axis_out] = -1
        wq = np.clip(np.round(w.astype(np.float64) / s_w.reshape(shape)), -127, 127).astype(np.int8)
        bq = np.round(bias.astype(np.float64) / (np.float64(s_in) * s_w)).astype(np.int64)
        bq = np.clip(bq, -(1 << 31), (1 << 31) - 1).astype(np.int32)
        ms = [quantize_multiplier(np.float64(s_in) * sw / np.float64(s_out)) for sw in s_w]
        q[prefix + "/w"] = wq
        q[prefix + "/bias"] = bq
        q[prefix + "/mult"] = np.asarray([m for m, _ in ms], np.int32)
        q[prefix + "/shift"] = np.asarray([s for _, s in ms], np.int32)

    w0 = tensors["first_conv/w"]
    conv_layer("q/first_conv", w0, np.zeros(w0.shape[2], np.float32), scales["in"], scales["c0"], 2)
    prev = "c0"
    for i in range(spec.n_blocks):
        d, pn = "d%d" % (i + 1), "p%d" % (i + 1)
        if identity[i]:
            # exact integer identity: weight 1 at weight scale 1, multiplier 1.0 = (2^30, shift 1), bias 0, same qparams in and out
            cin_i = tensors["b%d/dw/w" % i].shape[1]
            m1, s1 = quantize_multiplier(1.0)
            q["q/b%d/dw/w" % i] = np.ones((1, cin_i), np.int8)
            q["q/b%d/dw/bias" % i] = np.zeros(cin_i, np.int32)
            q["q/b%d/dw/mult" % i] = np.full(cin_i, m1, np.int32)
            q["q/b%d/dw/shift" % i] = np.full(cin_i, s1, np.int32)
        else:
            conv_layer("q/b%d/dw" % i, tensors["b%d/dw/w" % i], tensors["b%d/dw/b" % i], scales[prev], scales[d], 1)
        conv_layer("q/b%d/pw" % i, tensors["b%d/pw/w" % i], tensors["b%d/pw/b" % i], scales[d], scales[pn], 1)
        prev = pn
    # FULLY_CONNECTED: per-tensor symmetric weights
    hw = tensors["head/w"]
    s_w = float(np.abs(hw).max() / 127.0) or 1.0
    q["q/head/w"] = np.clip(np.round(hw.astype(np.float64) / s_w), -127, 127).astype(np.int8)
    q["q/head/bias"] = np.round(tensors["head/b"].astype(np.float64) / (np.float64(scales[prev]) * s_w)).astype(np.int32)
    m, sh = quantize_multiplier(np.float64(scales[prev]) * s_w / np.float64(scales["fc"]))
    q["q/head/mult"] = np.asarray([m], np.int32)
    q["q/head/shift"] = np.asarray([sh], np.int32)
    # LOGISTIC as the 256-entry table the builtin int8 kernel builds in float
    lut = np.zeros(256, np.int8)
    for v in range(-128, 128):
        x = np.float32(scales["fc"]) * np.float32(v - zps["fc"])
        y = np.float32(1.0) / (np.float32(1.0) + np.exp(-x, dtype=np.float32))
        r = np.round(np.float32(y * np.float32(256.0)))
        lut[v & 0xFF] = np.int8(np.clip(int(r) + zps["prob"], -128, 127))
    q["q/logistic_lut"] = lut
    return q


class StreamingInt8:
    """Integer streaming model.  Ring state holds int8 values initialised to the zero POINT of the
    tensor they buffer (real 0), not literal 0 (SURVEY.md Appendix C)."""

    def __init__(self, q: dict):
        self.q = q
        self.spec = Spec.decode(q["arch"])
        names = ["in", "c0"] + [n for i in range(self.spec.n_blocks) for n in ("d%d" % (i + 1), "p%d" % (i + 1))] + ["fc", "prob"]
        self.zp = dict(zip(names, [int(z) for z in q["q/zps"]]))
        self.scale = dict(zip(names, [np.float32(s) for s in q["q/scales"]]))
        self.reset()

    @property
    def input_scale(self):
        return self.scale["in"]

    @property
    def input_zero_point(self):
        return self.zp["in"]

    def reset(self):
        s = self.spec
        self.st_first = np.full((s.first_conv_kernel_size - 1 - (s.stride - 1), NUM_FEATURES), self.zp["in"], np.int8)
        self.st_block = []
        prev = "c0"
        for i in range(s.n_blocks):
            self.st_block.append(np.full((max(s.mixconv_kernel_sizes[i]) - 1, s.cin(i)), self.zp[prev], np.int8))
            prev = "p%d" % (i + 1)
        self.st_head = np.full((s.head_rows - 1, s.pointwise_filters[-1]), self.zp[prev], np.int8)

    def _requant(self, acc, prefix, zp_out, relu):
        y = mbqm(acc, self.q[prefix + "/mult"].astype(np.int64), self.q[prefix + "/shift"].astype(np.int64)) + zp_out
        lo = zp_out if relu else -128
        return np.clip(y, lo, 127).astype(np.int8)

    def step(self, x: np.ndarray, want_logit=False):
        """x: int8 [stride, 40] -> uint8 output value (0..255) as Python int."""
        s, q, zp = self.spec, self.q, self.zp
        x = np.asarray(x, np.int8).reshape(s.stride, NUM_FEATURES)
        mem = np.concatenate([self.st_first, x], 0)
        if self.st_first.shape[0]:
            self.st_first = mem[-self.st_first.shape[0]:]
        acc = np.einsum("kf,kfo->o", mem.astype(np.int64) - zp["in"], q["q/first_conv/w"].astype(np.int64)) + q["q/first_conv/bias"]
        net = self._requant(acc, "q/first_conv", zp["c0"], True)
        prev = "c0"
        for i in range(s.n_blocks):
            d, pn = "d%d" % (i + 1), "p%d" % (i + 1)
            mem = np.concatenate([self.st_block[i], net[None, :]], 0)
            if self.st_block[i].shape[0]:            # a 0-row ring (1-tap block) stays empty: mem[-0:] would be the whole window
                self.st_block[i] = mem[-self.st_block[i].shape[0]:]
            acc = ((mem.astype(np.int64) - zp[prev]) * q["q/b%d/dw/w" % i].astype(np.int64)).sum(0) + q["q/b%d/dw/bias" % i]
            dq = self._requant(acc, "q/b%d/dw" % i, zp[d], False)
            acc = (dq.astype(np.int64) - zp[d]) @ q["q/b%d/pw/w" % i].astype(np.int64) + q["q/b%d/pw/bias" % i]
            net = self._requant(acc, "q/b%d/pw" % i, zp[pn], True)
            prev = pn
        mem = np.concatenate([self.st_head, net[None, :]], 0)
        if self.st_head.shape[0]:                    # a 1-row head keeps no history: mem[-0:] would be the whole window
            self.st_head = mem[-self.st_head.shape[0]:]
        acc = ((mem.astype(np.int64) - zp[prev]) * q["q/head/w"].astype(np.int64)).sum() + int(q["q/head/bias"][0])
        logit = int(np.clip(mbqm(acc, int(q["q/head/mult"][0]), int(q["q/head/shift"][0])) + zp["fc"], -128, 127))
        if want_logit:
            return logit
        prob_i8 = int(q["q/logistic_lut"][logit & 0xFF])
        return prob_i8 + 128  # QUANTIZE int8 -> uint8 (inference_output_type uint8, utils.py:338)
