"""MWW model container (``.mww``): self-describing weight file for the streaming MixedNet.

The reference loads a ``.tflite`` flatbuffer at ``microwakeword/inference.py:36-45``.  No
TensorFlow / flatbuffers module and no ``.tflite`` file exist in this environment, so the
H100 build carries its own little-endian tensor container holding exactly what the
streaming graph needs (SURVEY.md section 7 step 2):

    0   char  magic[8]  = b"MWWB200\\0"
    8   u32   version   = 1
    12  u32   n_tensors
    16  u32   dir_offset
    20  u32   data_offset
    dir: n_tensors x { char name[48]; u32 dtype; u32 ndim; u32 shape[4]; u64 offset; u64 nbytes }
    data: raw arrays, each 64-byte aligned, offsets relative to the file start

The same bytes are handed to the C-ABI (``mww_create(blob, n, ...)``, include/mww.h), which
parses the directory in C++ -- no JSON, no Python objects cross the boundary.

Tensor naming (fp32 graph, BatchNorm folded as TFLite conversion does, utils.py:327-348):
    arch                 i32   MixedNet hyper-parameters (see ``Arch``; flag names mixednet.py:43-105)
    first_conv/w         f32   [kernel, 40, filters]       Conv2D(use_bias=False)  mixednet.py:317-329
    b{i}/dw/w            f32   [max_k, C] zero padded at the FRONT for the smaller MixConv kernels
                               (StridedKeep keeps the LAST k rows: strided_drop.py:80-84)
    b{i}/dw/ksize        i32   [C]   kernel size that owns each channel (mixednet.py:132-136)
    b{i}/dw/b            f32   [C]   DepthwiseConv2D default use_bias=True (mixednet.py:209-211)
    b{i}/pw/w, b{i}/pw/b f32   [Cin, Cout], [Cout]  1x1 conv + folded BN (mixednet.py:349-352)
    head/w, head/b       f32   [T_head, C], [1]     Flatten + Dense(1) (mixednet.py:383-384)
Integer graph (prefix ``q/``; TFLite int8 semantics, SURVEY.md Appendix C):
    q/scales f32[12], q/zps i32[12]  activation quant params in graph order
                                     [in, c0, d1, p1, d2, p2, d3, p3, d4, p4, fc, prob]
    q/<layer>/w i8, q/<layer>/bias i32, q/<layer>/mult i32, q/<layer>/shift i32
    q/logistic_lut i8[256]           indexed by the uint8 view of the int8 logit
"""

from __future__ import annotations

import dataclasses
import struct

import numpy as np

MAGIC = b"MWWB200\x00"
VERSION = 1
_DIR_ENTRY = struct.Struct("<48sII4IQQ")
_DTYPES = {0: np.float32, 1: np.int8, 2: np.int32, 3: np.uint8, 4: np.int16, 5: np.uint16}
_DTYPE_CODES = {np.dtype(v): k for k, v in _DTYPES.items()}

NUM_FEATURES = 40
FEATURE_SCALE = 0.0390625  # uint16 feature -> float, inference.py:94 / data.py:269


@dataclasses.dataclass(frozen=True)
class Arch:
    """MixedNet hyper-parameters; names follow the reference flags (mixednet.py:43-105)."""

    first_conv_filters: int = 32
    first_conv_kernel_size: int = 5
    stride: int = 3
    pointwise_filters: tuple = (64, 64, 64, 64)
    mixconv_kernel_sizes: tuple = ((5,), (7, 11), (9, 15), (23,))
    head_rows: int = 17  # time length of the final Stream(Identity) ring + 1 (mixednet.py:362-373)

    # ---- derived quantities (SURVEY.md Appendix A) ----
    @property
    def n_blocks(self) -> int:
        return len(self.pointwise_filters)

    def block_in_channels(self, i: int) -> int:
        return self.first_conv_filters if i == 0 else self.pointwise_filters[i - 1]

    def block_ring_rows(self, i: int) -> int:
        return max(self.mixconv_kernel_sizes[i]) - 1  # mixednet.py:193

    def channel_ksizes(self, i: int) -> np.ndarray:
        """Per-channel depthwise kernel size (_split_channels, mixednet.py:132-136)."""
        c = self.block_in_channels(i)
        ks = self.mixconv_kernel_sizes[i]
        split = [c // len(ks)] * len(ks)
        split[0] += c - sum(split)
        return np.concatenate([np.full(n, k, np.int32) for n, k in zip(split, ks)])

    @property
    def first_conv_ring_rows(self) -> int:
        # stream.py:253-255: max(0, dilation*(k-1) - (stride-1))
        return max(0, self.first_conv_kernel_size - 1 - (self.stride - 1))

    @property
    def state_elements(self) -> int:
        n = self.first_conv_ring_rows * NUM_FEATURES
        for i in range(self.n_blocks):
            n += self.block_ring_rows(i) * self.block_in_channels(i)
        n += (self.head_rows - 1) * self.pointwise_filters[-1]
        return n

    @property
    def macs_per_step(self) -> int:
        n = self.first_conv_kernel_size * NUM_FEATURES * self.first_conv_filters
        for i in range(self.n_blocks):
            n += int(self.channel_ksizes(i).sum())
            n += self.block_in_channels(i) * self.pointwise_filters[i]
        n += self.head_rows * self.pointwise_filters[-1]
        return n

    def encode(self) -> np.ndarray:
        v = [self.first_conv_filters, self.first_conv_kernel_size, self.stride, NUM_FEATURES,
             self.n_blocks, self.head_rows]
        for f, ks in zip(self.pointwise_filters, self.mixconv_kernel_sizes):
            if len(ks) > 4:
                raise ValueError("at most 4 MixConv kernel sizes per block")
            v += [f, len(ks)] + list(ks) + [0] * (4 - len(ks))
        return np.asarray(v, np.int32)

    @staticmethod
    def decode(v: np.ndarray) -> "Arch":
        v = [int(x) for x in v]
        if v[3] != NUM_FEATURES:
            raise ValueError("model expects %d features per row, this build has 40" % v[3])
        nb = v[4]
        pw, ks = [], []
        for b in range(nb):
            o = 6 + 6 * b
            pw.append(v[o])
            ks.append(tuple(v[o + 2:o + 2 + v[o + 1]]))
        return Arch(v[0], v[1], v[2], tuple(pw), tuple(ks), v[5])


OKAY_NABU = Arch()  # notebooks/basic_training_notebook.ipynb:503-509

# activation tensor order of q/scales, q/zps
def act_names(arch: Arch):
    names = ["in", "c0"]
    for i in range(arch.n_blocks):
        names += ["d%d" % (i + 1), "p%d" % (i + 1)]
    return names + ["fc", "prob"]


def write_container(tensors: dict) -> bytes:
    """Serialise ``{name: ndarray}`` (must include ``arch``) to container bytes."""
    if "arch" not in tensors:
        raise ValueError("container needs an 'arch' tensor")
    names = list(tensors)
    dir_offset = 24
    data_offset = dir_offset + _DIR_ENTRY.size * len(names)
    data_offset = (data_offset + 63) // 64 * 64
    entries, blobs, cursor = [], [], data_offset
    for name in names:
        a = np.ascontiguousarray(tensors[name])
        if a.dtype not in _DTYPE_CODES:
            raise TypeError("%s: unsupported dtype %s" % (name, a.dtype))
        if a.ndim > 4 or len(name.encode()) > 47:
            raise ValueError("%s: rank > 4 or name too long" % name)
        shape = list(a.shape) + [1] * (4 - a.ndim)
        raw = a.astype(a.dtype.newbyteorder("<")).tobytes()
        entries.append(_DIR_ENTRY.pack(name.encode(), _DTYPE_CODES[a.dtype], a.ndim, *shape, cursor, len(raw)))
        pad = (-len(raw)) % 64
        blobs.append(raw + b"\0" * pad)
        cursor += len(raw) + pad
    head = MAGIC + struct.pack("<IIII", VERSION, len(names), dir_offset, data_offset)
    body = head + b"".join(entries)
    body += b"\0" * (data_offset - len(body))
    return body + b"".join(blobs)


def read_container(blob: bytes) -> dict:
    """Parse container bytes to ``{name: ndarray}``; raises ValueError on a malformed file."""
    if len(blob) < 24 or blob[:8] != MAGIC:
        raise ValueError("not an MWW model container (bad magic)")
    version, n, dir_offset, data_offset = struct.unpack_from("<IIII", blob, 8)
    if version != VERSION:
        raise ValueError("unsupported container version %d" % version)
    out = {}
    for i in range(n):
        name, dt, ndim, s0, s1, s2, s3, off, nbytes = _DIR_ENTRY.unpack_from(blob, dir_offset + i * _DIR_ENTRY.size)
        if dt not in _DTYPES or ndim > 4 or off + nbytes > len(blob) or off < data_offset:
            raise ValueError("corrupt directory entry %d" % i)
        shape = (s0, s1, s2, s3)[:ndim]
        a = np.frombuffer(blob, dtype=np.dtype(_DTYPES[dt]).newbyteorder("<"), count=nbytes // np.dtype(_DTYPES[dt]).itemsize, offset=off)
        out[name.rstrip(b"\0").decode()] = a.reshape(shape).astype(_DTYPES[dt])
    return out


def load(path: str) -> dict:
    with open(path, "rb") as f:
        return read_container(f.read())


def save(path: str, tensors: dict) -> None:
    with open(path, "wb") as f:
        f.write(write_container(tensors))


def is_quantized(tensors: dict) -> bool:
    return "q/scales" in tensors
