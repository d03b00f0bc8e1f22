"""Plan for running the reference's sequential, state-carrying evaluation loop as one batched pass.

The reference's harness (microwakeword/test.py:293-517) calls ``Model.predict_spectrogram`` once per track on one
interpreter that is never reset, so the steps of all tracks form one sequence fed to one model.  A streaming MixedNet
keeps a finite history: after ``warmup_steps(arch)`` steps from ANY starting state, every ring holds only values
computed from the rows fed during those steps.  So the sequence can be cut into S contiguous segments of L steps and
segment i run on stream i of a batched engine, provided stream i is first fed the W = stride * warmup_steps rows that
precede its segment (outputs discarded).  Stream 0 takes the model's current state instead of a warm-up.  The
probabilities come out row-major [S, L], which is the global step sequence; track k is the slice at its cumulative step
offset.  ``Model.predict_spectrograms`` carries this out; ``plan`` is the pure, host-only part of it.
"""

from __future__ import annotations

import dataclasses

import numpy as np


def warmup_steps(arch) -> int:
    """Model steps after which the state no longer depends on the state before them (``model_file.Arch``):
    ceil(first_conv_ring_rows / stride) steps refill the first-conv ring from fed rows, each block ring then needs
    block_ring_rows(b) steps of clean outputs from the layer below, and the head ring head_rows - 1 more.
    67 steps (201 rows) for okay_nabu."""
    first = -(-arch.first_conv_ring_rows // arch.stride)
    return first + sum(arch.block_ring_rows(b) for b in range(arch.n_blocks)) + arch.head_rows - 1


@dataclasses.dataclass(frozen=True)
class Plan:
    n_streams: int            # S: segments = streams of the batched engine
    seg_steps: int            # L: model steps per segment (the last one is padded up to L)
    warmup_steps: int         # model steps fed before each segment after the first
    total_steps: int          # N: real steps of all tracks together
    track_offsets: np.ndarray  # int64 [n_tracks]: first step of each track in the [S, L] row-major output

    @property
    def last_segment_steps(self) -> int:
        """Real steps in the last segment (1 .. L; 0 only when there are no steps at all)."""
        return self.total_steps - (self.n_streams - 1) * self.seg_steps


def plan(step_counts, stride: int, warmup_rows: int, max_streams: int = 65536) -> Plan:
    """(per-track step counts, rows per step, warm-up rows W, stream cap) -> Plan.

    Rule: S = clamp(N // (4 * W_steps), 1, max_streams) with W_steps = ceil(W / stride), then L = ceil(N / S), and S is
    lowered to ceil(N / L) so that no segment is empty.  Warm-up work is then at most a quarter of the real work, and
    S > 1 implies L >= 4 * W_steps >= W_steps: a segment is always at least as long as the warm-up it needs, so the
    warm-up rows of segment i lie inside segment i - 1 (they are the real rows just before segment i).  N < 4 * W_steps
    gives S = 1: one call on the model's own engine, no warm-up."""
    steps = np.asarray(step_counts, np.int64).reshape(-1)
    if (steps < 0).any():
        raise ValueError("step counts must be >= 0")
    if stride < 1 or warmup_rows < 0 or max_streams < 1:
        raise ValueError("stride and max_streams must be >= 1, warmup_rows >= 0")
    w_steps = -(-int(warmup_rows) // int(stride))
    offsets = np.zeros(steps.size, np.int64)
    if steps.size > 1:
        offsets[1:] = np.cumsum(steps[:-1])
    n = int(steps.sum())
    if n == 0:
        return Plan(1, 0, w_steps, 0, offsets)
    s = min(max(n // (4 * max(w_steps, 1)), 1), int(max_streams))
    seg = -(-n // s)
    s = -(-n // seg)
    return Plan(s, seg, w_steps, n, offsets)
