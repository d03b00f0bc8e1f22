"""The wgmma clip kernel's scheduling cases (run with -m gpu on an H100).

nn_f32_clip_tc_kernel runs min(streams, 2 x SMs) persistent CTAs.  Inside a CTA each warpgroup produces and contracts its own 64
steps of a chunk, the two meet at the shared weight buffers (refilled by whichever warpgroup finishes a slot last, including the
next chunk's first two slots), and each block's input ring is staged from the stream's state one block ahead.  The cases here
are the ones that scheduling creates: CTAs with no stream or one stream more than their neighbours, chunks where one warpgroup
has no steps (n <= 64) or only a few, calls entering with 0, 1 and 2 pending rows, and ring state that a previous stream, call
or reset left behind.

Inputs follow tests/test_gpu_full_size.py: P_ROWS distinct base streams (prime), stream s carries base[s % P]."""

import numpy as np
import pytest

import oracle
from test_gpu_full_size import F32_TOL, P_ROWS, _base_audio, _blob, check_streams, periodic_streams

pytestmark = pytest.mark.gpu

# rows per call and the steps they give: (pending + rows) // 3, entering with the pending rows the previous call left
CALLS = [49, 189, 192, 196, 379, 385, 387, 772, 190, 191, 47]
STEPS = [16, 63, 64, 65, 127, 128, 129, 257, 64, 63, 16]
PENDING_IN = [0, 1, 1, 1, 2, 0, 1, 1, 2, 0, 2]


@pytest.fixture(scope="module")
def rows_and_oracle():
    total = sum(CALLS)
    audio = _base_audio(P_ROWS, 480 + 160 * (total - 1), 9100)
    feats, want = oracle.run_pipeline(_blob("okay_nabu_synth_f32.mww"), audio, threads=8)
    assert feats.shape == (P_ROWS, total, 40) and want.shape == (P_ROWS, total // 3)
    return feats, want


def _stream_counts(sms):
    # 1 stream; one CTA idle; one CTA with a second stream; 5 x SMs + 7: a third wave in which only 7 of the 2 x SMs CTAs work
    return [1, 2 * sms - 1, 2 * sms + 1, 5 * sms + 7]


@pytest.mark.parametrize("which", range(4))
def test_uneven_stream_counts_through_chunk_boundaries(torch_cuda, rows_and_oracle, which):
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    feats, want = rows_and_oracle
    S = _stream_counts(torch.cuda.get_device_properties(0).multi_processor_count)[which]
    rows = periodic_streams(torch, feats, S, ())
    eng = StreamEngine(_blob("okay_nabu_synth_f32.mww"), n_streams=S)
    got, pos = [], 0
    for r, steps, pend in zip(CALLS, STEPS, PENDING_IN):
        assert eng.pending_rows == pend
        out = eng.infer(rows.view(torch.int16)[:, pos:pos + r].contiguous().view(torch.uint16))
        assert out.shape == (S, steps), (r, out.shape)
        got.append(out)
        pos += r
    got = torch.cat(got, 1)
    if S >= P_ROWS:
        check_streams(torch, got, want, False, "S=%d" % S)
    else:
        err = np.abs(got.cpu().numpy() - want[:S, :got.shape[1]]).max()
        assert err <= F32_TOL, (S, err)


def test_clip_and_live_calls_with_partial_resets(torch_cuda, rows_and_oracle):
    """Clip calls (wgmma kernel) alternate with one-step calls (live kernel) and a reset of every fifth stream, taken with no
    rows pending: the reset streams must start from zero rings, the others must carry on, whatever ring a CTA staged before."""
    from microwakeword_b200.engine import StreamEngine
    torch = torch_cuda
    feats, want = rows_and_oracle
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = 6 * sms + 37                                  # >= 3 streams per CTA, a partial last wave
    blob = _blob("okay_nabu_synth_f32.mww")
    rows = periodic_streams(torch, feats, S, ("clip_tc",))
    eng = StreamEngine(blob, n_streams=S)
    plan = [300, 3, 3, 3, 3, 387, "reset", 200, 3, 3, 196, 3, 385]
    before, after, pos, pos_reset = [], [], 0, None
    for r in plan:
        if r == "reset":
            assert eng.pending_rows == 0
            eng.reset(list(range(0, S, 5)))
            pos_reset = pos
            continue
        out = eng.infer(rows.view(torch.int16)[:, pos:pos + r].contiguous().view(torch.uint16))
        (before if pos_reset is None else after).append(out)
        pos += r
    before, after = torch.cat(before, 1), torch.cat(after, 1)
    n0 = before.shape[1]
    assert n0 == pos_reset // 3
    check_streams(torch, before, want, False, "before the reset")
    # streams that were not reset carry on as one long call; reset ones restart from zero rings on the rows after the reset
    net = oracle.MixedNet(blob)
    fresh = []
    for b in range(P_ROWS):
        net.reset()
        fresh.append(net.predict_u16(feats[b, pos_reset:pos]))
    fresh = np.stack(fresh)
    assert fresh.shape[1] == after.shape[1]
    got = after.cpu().numpy()
    ids = np.arange(S)
    reset = ids % 5 == 0
    bits = got.view(np.int32)
    for mask, ref in ((reset, fresh), (~reset, want[:, n0:n0 + got.shape[1]])):
        sel = ids[mask]
        err = np.abs(got[sel] - ref[sel % P_ROWS]).max()
        assert err <= F32_TOL, (err, "reset" if mask is reset else "carried")
        # streams with the same content and the same history agree bit for bit
        first = {}
        for s in sel:
            k = s % P_ROWS
            if k in first:
                assert np.array_equal(bits[s], bits[first[k]]), (s, first[k])
            else:
                first[k] = s
