"""A third, independent reading of the reference's MixedNet graph for the (otherwise unpinned) NN oracle.

`oracle/mixednet_ref.py` and `oracle/mixednet.c` are hand-written loops.  Here the NON-STREAMING Keras graph of
microwakeword/mixednet.py:278-386 is restated layer by layer with PyTorch's own convolution operators on the KERAS-form
parameters (BatchNorm not folded, MixConv groups as separate depthwise convs, `StridedDrop` alignment as in
mixednet.py:222-224), and its logits must agree with the oracle's non-streaming and streaming forms.  What this guards:
conv orientation (cross-correlation, oldest tap first), Keras kernel layouts, the `_split_channels` rule
(mixednet.py:132-136), "the shorter kernel sees the LAST k rows", BatchNorm folding (epsilon 1e-3) and the Flatten order
of the head.  It cannot pin TensorFlow's arithmetic itself -- no TensorFlow exists here (DESIGN.md section 0)."""

import numpy as np
import pytest

from oracle import mixednet_ref as R

torch = pytest.importorskip("torch")
F = torch.nn.functional

SPECS = {
    "okay_nabu": R.Spec(),
    "stride2_three_groups": R.Spec(16, 6, 2, (40,), ((7, 11, 13),), head_rows=9),
    "uneven_split": R.Spec(20, 4, 1, (50, 30), ((3, 5, 7), (5, 9)), head_rows=4),       # 50 channels / 3 groups -> 18, 16, 16
    "block_without_mixconv": R.Spec(24, 6, 2, (32, 16, 24), ((3, 5), (1,), (7,)), head_rows=4),   # mixednet.py:346-348
    "one_row_head": R.Spec(32, 6, 3, (48, 24), ((3,), (5,)), head_rows=1),                  # the head keeps no history
}


def keras_graph_logits(spec, p, x):
    """x: float32 [T, 40] -> logits for every position with a full receptive field, float64 throughout."""
    t = torch.from_numpy(np.asarray(x, np.float64)).T[None]                               # [1, 40, T]: features are the conv channels
    w0 = torch.from_numpy(p["first_conv/kernel"].astype(np.float64)).permute(2, 1, 0)     # Keras (k, in, out) -> (out, in, k)
    net = torch.relu(F.conv1d(t, w0, stride=spec.stride))                                 # Conv2D((k0, 1), strides=(stride, 1), 'valid', no bias) + ReLU
    for i in range(spec.n_blocks):
        ks = spec.mixconv_kernel_sizes[i]
        if max(ks) > 1:                                                                     # mixednet.py:346-348: otherwise no MixConv layer at all
            splits = [net.shape[1] // len(ks)] * len(ks)
            splits[0] += net.shape[1] - sum(splits)                                        # _split_channels
            outs = []
            for xs, k, kern, bias in zip(torch.split(net, splits, dim=1), ks, p["b%d/dw/kernels" % i], p["b%d/dw/biases" % i]):
                w = torch.from_numpy(kern.astype(np.float64)).T[:, None, :]                # Keras (k, channels) -> (channels, 1, k)
                outs.append(F.conv1d(xs, w, torch.from_numpy(bias.astype(np.float64)), groups=xs.shape[1]))   # DepthwiseConv2D((k, 1), 'valid')
            keep = outs[-1].shape[2]
            outs = [o[:, :, o.shape[2] - keep:] for o in outs]                              # StridedDrop: drop the EARLIEST rows
            net = torch.cat(outs, 1)
        pw = torch.from_numpy(p["b%d/pw/kernel" % i].astype(np.float64)).T[:, :, None]     # (in, out) -> (out, in, 1)
        net = F.conv1d(net, pw)                                                             # Conv2D(filters, 1, no bias)
        g, b = (torch.from_numpy(p["b%d/bn/%s" % (i, n)].astype(np.float64))[None, :, None] for n in ("gamma", "beta"))
        m, v = (torch.from_numpy(p["b%d/bn/%s" % (i, n)].astype(np.float64))[None, :, None] for n in ("mean", "var"))
        net = torch.relu(g * (net - m) / torch.sqrt(v + 1e-3) + b)                          # BatchNormalization (inference) + ReLU
    dense = torch.from_numpy(p["dense/kernel"].astype(np.float64)).reshape(spec.head_rows, net.shape[1])   # Flatten of [time, 1, channel]
    win = net[0].T.unfold(0, spec.head_rows, 1).permute(0, 2, 1)                            # [positions, head_rows, channels]
    return ((win * dense[None]).sum((1, 2)) + float(p["dense/bias"][0])).numpy()


@pytest.mark.parametrize("name", list(SPECS))
def test_oracle_forms_equal_the_keras_graph_built_from_library_convolutions(name):
    spec = SPECS[name]
    p = R.init_synthetic(spec, seed=3)
    folded = R.fold_bn(spec, p)
    rng = np.random.default_rng(5)
    s = spec.stride
    field = spec.first_conv_kernel_size + s * (sum(max(k) - 1 for k in spec.mixconv_kernel_sizes) + spec.head_rows - 1)
    T = field + 11 * s
    x = rng.uniform(0, 26, (T, 40)).astype(np.float32)
    want = keras_graph_logits(spec, p, x)
    assert want.shape == (12,)
    # (1) the oracle's non-streaming form on the folded tensors
    ns = R.nonstreaming_logits(folded, x)
    assert ns.shape == want.shape and np.abs(ns - want).max() < 2e-4 * max(1.0, np.abs(want).max())
    # (2) the oracle's STREAMING form.  Its first conv sees ring0 = k0 - stride rows of (zero) history before the first real
    # row, so step j reads rows [j s - ring0, j s + s) of what it is fed; feeding x[ring0 % s:] puts step j on the
    # non-streaming first-conv position j - ring0 // s, and the logit of position q is the step whose newest first-conv
    # output is q + span (span = every later ring's length).  All rows that position uses are real ones.
    m = R.FoldedStreamingF32(folded)
    ring0 = spec.first_conv_kernel_size - s
    span = sum(max(k) - 1 for k in spec.mixconv_kernel_sizes) + spec.head_rows - 1
    xs = x[ring0 % s:]
    n_steps = xs.shape[0] // s
    logits = np.asarray([m.step(xs[j * s:(j + 1) * s], want_logit=True) for j in range(n_steps)])
    offs = [q + span + ring0 // s for q in range(len(want))]
    assert all(0 <= o < n_steps for o in offs)
    assert np.abs(logits[offs] - want).max() < 2e-4 * max(1.0, np.abs(want).max())
    assert np.std(want) > 1e-3
