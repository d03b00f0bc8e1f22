"""Geometries across the range mww_create accepts for the run-time-geometry MixedNet (mww_nn_generic.cuh), their models,
and the float64 error-bound check -- shared by tests/test_generic_range.py (CPU, host emulation of the phase functions)
and tests/test_zz_generic_range_gpu.py (the kernels through the C-ABI).  TEST INFRASTRUCTURE."""

import functools

import numpy as np

import oracle
from host_emul import emul
from microwakeword_b200.synth_audio import synth_audio
from oracle import mixednet_ref as R

GEOMETRIES = {
    # 4 channel passes of the 128-thread loops; 257 and 129 are one channel past a pass; 4 uneven MixConv groups; a 1-tap
    # group inside a block; 52.3 KiB of shared memory (above the 48 KiB that needs the opt-in)
    "wide": R.Spec(512, 5, 3, (257, 129, 512), ((3, 5, 7, 9), (1, 11), (5,)), head_rows=8),
    # 8 blocks, 64-tap first conv at stride 1, 64-tap rings in five blocks, a 64-row head: 169 KiB, one CTA per SM
    "deep": R.Spec(96, 64, 1, (96,) * 8, ((64,), (3, 64), (5,), (64, 7, 9, 11), (1,), (64,), (33, 2), (64,)), head_rows=64),
    # stride > 16: up to 16 pending rows
    "long_stride": R.Spec(24, 40, 17, (48, 32), ((5, 9), (3,)), head_rows=6),
    # k0 = stride = 64: no first-conv ring, up to 63 pending rows
    "max_stride": R.Spec(16, 64, 64, (32,), ((3,),), head_rows=2),
    # no ring anywhere (state_elems == 0): 1-tap blocks and a 1-row head
    "stateless": R.Spec(32, 3, 3, (48, 24), ((1,), (1,)), head_rows=1),
}

SMEM_CAP = 200 * 1024               # bytes of shared memory one stream of the generic kernels may use


def boundary_base(last_cout, head_rows):
    return R.Spec(64, 5, 3, (512, last_cout), ((9,), (53, 3)), head_rows=head_rows)


@functools.lru_cache(maxsize=None)
def boundary_specs():
    """{4-byte shared-memory elements: Spec} for 51 200 (exactly 200 KiB) and 51 201 (4 bytes over), found by searching
    (last cout, head_rows) of boundary_base with the kernels' own geometry function"""
    found = {}
    for x in range(1, 513):
        for h in range(1, 65):
            info = emul.gen_arch_info(boundary_base(x, h).encode())
            if info["rc"] == 0 and info["sm_elems"] in (SMEM_CAP // 4, SMEM_CAP // 4 + 1):
                found.setdefault(info["sm_elems"], (x, h))
    return {k: boundary_base(*v) for k, v in found.items()}


def all_geometries():
    g = dict(GEOMETRIES)
    g["boundary"] = boundary_specs()[SMEM_CAP // 4]
    return g


def features(n_streams, n_samples, seed):
    audio = np.stack([synth_audio(n_samples, seed + i) for i in range(n_streams)])
    feats, _ = oracle.run_pipeline(None, audio, want_probs=False)
    return feats                                                     # uint16 [S, T, 40]


@functools.lru_cache(maxsize=None)
def _models_cached(key):
    spec = R.Spec.decode(np.asarray(key, np.int32))
    f32 = R.fold_bn(spec, R.init_synthetic(spec, 0))
    rows = max(200, 20 * spec.stride)
    calib = features(1, rows * 160, 7000).reshape(-1, 40)
    calib = calib[: calib.shape[0] // spec.stride * spec.stride].reshape(-1, spec.stride, 40)
    return f32, R.quantize_model(f32, calib.astype(np.float32) * R.FEATURE_SCALE)


def models(spec):
    """(fp32 container tensors, int8 container tensors) of `spec`: synthetic weights, int8 calibrated on synthetic audio"""
    return _models_cached(tuple(int(v) for v in spec.encode()))


def call_cuts(stride, n_rows):
    """a ragged split of n_rows rows: a call of 1 row, calls with no full step, a call that leaves stride - 1 rows pending"""
    s = stride
    return sorted({c for c in (0, 1, 2, s - 1, 2 * s - 1, 2 * s + 3, 3 * s + 3, n_rows // 2, n_rows - 1, n_rows) if 0 <= c <= n_rows})


def f64_run(f32_tensors, rows_u16):
    """StreamingF64 over whole steps of one stream's uint16 rows -> (p64, bound on p, ring values, ring bounds)"""
    m = R.StreamingF64(f32_tensors)
    s = m.spec.stride
    x = rows_u16.astype(np.float32) * R.FEATURE_SCALE
    out = [m.step(x[j:j + s]) for j in range(0, x.shape[0] // s * s, s)]
    p = np.asarray([o[0] for o in out])
    e = np.asarray([o[1] for o in out])
    vals, errs = m.state()
    return p, e, vals, errs


RING_RTOL = 1e-5                    # fp32 ring entries against the float64 values: |got - v| <= RING_RTOL * max(1, |v|)


def ring_tolerance_violations(got, vals):
    """entries of an fp32 ring state further than RING_RTOL * max(1, |v|) from the float64 values -- a check that does not
    depend on the running bound, which is a worst case and grows with depth"""
    got, vals = np.asarray(got, np.float64).ravel(), np.asarray(vals, np.float64).ravel()
    return int(np.count_nonzero(np.abs(got - vals) > RING_RTOL * np.maximum(1.0, np.abs(vals))))


def bound_tightness(f32_tensors, rows_u16):
    """how tight the float64 bound is after one stream's rows: {ring: median bound / |value|} over the computed nonzero
    entries of every block ring ("b<i>", absent for a 1-tap block) and the head ring, and the median of bound / p over the
    probabilities ("prob")"""
    m = R.StreamingF64(f32_tensors)
    s = m.spec.stride
    x = rows_u16.astype(np.float32) * R.FEATURE_SCALE
    steps = [m.step(x[j:j + s]) for j in range(0, x.shape[0] // s * s, s)]
    out = {"prob": float(np.median([e / p for p, e, _, _ in steps]))}
    for name, v, e in [("b%d" % i, r, er) for i, (r, er) in enumerate(zip(m.st_block, m.e_block))] + [("head", m.st_head, m.e_head)]:
        v, e = np.abs(v).ravel(), e.ravel()
        nz = (v > 0) & (e > 0)
        if nz.any():
            out[name] = float(np.median(e[nz] / v[nz]))
    return out


def bound_violations(got, want, bound):
    """(number of elements outside the bound, median of bound / |value| over the computed nonzero values -- exact inputs
    carry a zero bound and are left out)"""
    got, want, bound = (np.asarray(a, np.float64).ravel() for a in (got, want, bound))
    bad = int(np.count_nonzero(np.abs(got - want) > bound))
    nz = (np.abs(want) > 0) & (bound > 0)
    return bad, float(np.median(bound[nz] / np.abs(want[nz]))) if nz.any() else 0.0
