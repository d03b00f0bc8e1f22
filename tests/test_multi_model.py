"""Several models over one frontend, the parts that need no GPU: the C-ABI refuses an empty model list and fails loudly
without a device, and the host-side step / shape bookkeeping (engine.call_plan) for models of different strides agrees
with counting the frontend's windows one sample at a time."""

import os

import numpy as np
import pytest

from conftest import GOLDEN


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on GPU-less hosts")
    from microwakeword_b200 import _lib
    from microwakeword_b200.engine import MultiModelEngine
    f32 = os.path.join(GOLDEN, "okay_nabu_synth_f32.mww")
    i8 = os.path.join(GOLDEN, "okay_nabu_synth_int8.mww")
    with pytest.raises(_lib.MwwError) as e:
        MultiModelEngine([f32, i8], n_streams=4)
    assert e.value.code == -3 and "no CUDA device" in str(e.value)


def test_an_empty_model_list_is_refused_before_any_device_work():
    from microwakeword_b200 import _lib
    from microwakeword_b200.engine import MultiModelEngine
    with pytest.raises(_lib.MwwError) as e:
        MultiModelEngine([], n_streams=4)
    assert e.value.code == -1 and "n_models" in str(e.value)
    with pytest.raises(ValueError):
        MultiModelEngine([None], n_streams=4)


def _windows(total_samples, hop):
    """windows of 480 samples every `hop` samples that fit in the first total_samples samples"""
    return max((total_samples - 480) // hop + 1, 0)


@pytest.mark.parametrize("hop", [160, 320, 16, 480])
def test_call_plan_counts_rows_and_steps_per_stride(hop):
    from microwakeword_b200.engine import call_plan
    strides = [3, 17, 1, 64, 3]
    rng = np.random.default_rng(hop)
    calls = [480, 0, 479, 1, 48000, 47999, 48001] + [int(v) for v in rng.integers(0, 5000, 40)] + [480] * 20
    buffered, pending = 0, [0] * len(strides)
    seen, rows_total, steps_total = 0, 0, [0] * len(strides)
    for n in calls:
        rows, steps, buffered_after, pending_after = call_plan(buffered, n, hop, pending, strides)
        seen += n
        assert rows == _windows(seen, hop) - rows_total                      # what the frontend emits for this call
        rows_total += rows
        assert buffered_after == seen - rows_total * hop and 0 <= buffered_after < 480 + hop
        for k, s in enumerate(strides):
            steps_total[k] += steps[k]
            assert steps_total[k] == rows_total // s and pending_after[k] == rows_total % s
        buffered, pending = buffered_after, pending_after
    assert steps_total[0] == steps_total[4] and steps_total[2] == rows_total


def test_call_plan_of_one_model_is_the_single_engine_rule():
    from microwakeword_b200.engine import call_plan, rows_for
    for buffered in (0, 1, 159, 320, 479):
        for n in (0, 1, 160, 480, 47999, 48000):
            for pend, stride in ((0, 3), (2, 3), (16, 17)):
                rows, steps, _, _ = call_plan(buffered, n, 160, [pend], [stride])
                assert rows == rows_for(buffered, n, 160)
                assert steps == [(pend + rows) // stride]
