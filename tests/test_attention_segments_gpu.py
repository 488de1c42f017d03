"""GPU: segment-masked causal attention (fsb_sdpa_fwd_segments / fsb_sdpa_bwd_segments, ops.sdpa_segments_*) for packed rows.

Each segment of a packed row is an independent causal attention, so every segment is checked against the fp64 bounds of the
causal launch checkers (tests/launch_refs.py verify_sdpa_fwd / verify_sdpa_bwd) run on that segment's slices alone. Exact
answers: one segment per row is the causal kernel bit for bit; one-token segments give O == V and dV == dO. Tile skipping:
NaN planted in one segment's operands never reaches another segment, which masking alone could not achieve (a loaded NaN
reaches the MMA)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import launch_refs as R  # noqa: E402
from fsb200 import ops  # noqa: E402

DEV = "cuda"


def _rows_from_lengths(layouts, S):
    """segment_ids [B, S] from per-row segment lengths (a short sum leaves a trailing pad segment)."""
    ids = torch.zeros((len(layouts), S), dtype=torch.int64)
    for b, lens in enumerate(layouts):
        t = 0
        for k, n in enumerate(lens):
            ids[b, t:t + n] = k
            t += n
        assert t <= S
        ids[b, t:] = len(lens)
    return ids


def _random_lengths(S, seed, pad=37):
    """Two one-token segments, then seeded lengths in [1, 300) up to S - pad: the rest of the row is a pad segment."""
    g = torch.Generator().manual_seed(seed)
    lens, t = [1, 1], 2
    while t < S - pad:
        n = min(int(torch.randint(1, 300, (1,), generator=g)), S - pad - t)
        lens.append(n)
        t += n
    return lens


def _segments(seg_ids):
    """Per row the list of (start, end) runs."""
    out = []
    for row in seg_ids.tolist():
        runs, s = [], 0
        for t in range(1, len(row) + 1):
            if t == len(row) or row[t] != row[t - 1]:
                runs.append((s, t))
                s = t
        out.append(runs)
    return out


def _qkv(B, S, H, D, seed):
    """q / k / v as strided views of a per-head interleaved packed QKV buffer (the LLaMA layout)."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, S, H, 3, D, generator=g).to(torch.bfloat16).to(DEV)
    return qkv, (qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2])


def _run(qkv, seg_ids, D, seed):
    B, S, H = qkv.shape[:3]
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    scale = 1.0 / math.sqrt(D)
    st, en = ops.segment_bounds(seg_ids.to(DEV))
    out, lse = ops.sdpa_segments_fwd(q, k, v, scale, st, en)
    g = torch.Generator().manual_seed(seed + 1)
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(DEV)
    dqkv = torch.full_like(qkv, float("nan"))
    ops.sdpa_segments_bwd(q, k, v, out, dout, lse, scale, st, en, dqkv[:, :, :, 0], dqkv[:, :, :, 1], dqkv[:, :, :, 2])
    torch.cuda.synchronize()
    return out, lse, dout, dqkv


def _verify(qkv, seg_ids, out, lse, dout, dqkv, D, rows=None, only=None):
    """fp64 bounds on every segment (or the segments `only(b, s, e)` accepts) of the given rows."""
    scale = 1.0 / math.sqrt(D)
    bound = R.Bound("segments")
    for b, runs in enumerate(_segments(seg_ids)):
        if rows is not None and b not in rows:
            continue
        for s, e in runs:
            if only is not None and not only(b, s, e):
                continue
            sl = lambda t: t[b:b + 1, s:e]
            q, k, v = (sl(qkv[:, :, :, i]) for i in range(3))
            R.verify_sdpa_fwd(bound, q, k, v, scale, True, None, None, sl(out), lse[b:b + 1, :, s:e], None)
            R.verify_sdpa_bwd(bound, q, k, v, sl(out), sl(dout), lse[b:b + 1, :, s:e], scale, True,
                              sl(dqkv[:, :, :, 0]), sl(dqkv[:, :, :, 1]), sl(dqkv[:, :, :, 2]))
    return bound


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("S", [128, 200, 1024, 2048])
def test_segments_vs_fp64(S, D):
    """Seeded random lengths with one-token segments and a trailing pad segment in row 0; row 1 a different layout."""
    layouts = [_random_lengths(S, seed=S + D), [S // 2, S - S // 2 - 5, 5]]
    seg_ids = _rows_from_lengths(layouts, S)
    qkv, _ = _qkv(2, S, 2, D, seed=S)
    out, lse, dout, dqkv = _run(qkv, seg_ids, D, seed=S)
    assert not torch.isnan(dqkv.float()).any(), "unwritten gradient elements"
    _verify(qkv, seg_ids, out, lse, dout, dqkv, D)


@pytest.mark.parametrize("D", [64, 128])
def test_segments_at_tile_boundaries(D):
    """Segment edges at 63 / 64 / 65 and 127 / 128 / 129 (the 64-row streamed tiles and 128-row resident tiles)."""
    S = 1024
    layouts = [[63, 1, 65, 127, 1, 129, 128, 64], [64, 64, 129, 127, 128, 65, 63], [128, 128, 256, 512]]
    seg_ids = _rows_from_lengths(layouts, S)
    qkv, _ = _qkv(3, S, 2, D, seed=7)
    out, lse, dout, dqkv = _run(qkv, seg_ids, D, seed=7)
    _verify(qkv, seg_ids, out, lse, dout, dqkv, D)


@pytest.mark.parametrize("S", [256, 200])
@pytest.mark.parametrize("D", [64, 128])
def test_one_segment_is_the_causal_kernel_bit_for_bit(S, D):
    qkv, (q, k, v) = _qkv(2, S, 2, D, seed=3)
    scale = 1.0 / math.sqrt(D)
    seg_ids = torch.zeros((2, S), dtype=torch.int64)
    out, lse, dout, dqkv = _run(qkv, seg_ids, D, seed=3)
    o_c, lse_c = ops.sdpa_fwd(q, k, v, scale, True)
    d_c = torch.empty_like(qkv)
    ops.sdpa_bwd(q, k, v, o_c, dout, lse_c, scale, True, d_c[:, :, :, 0], d_c[:, :, :, 1], d_c[:, :, :, 2])
    torch.cuda.synchronize()
    assert torch.equal(out, o_c) and torch.equal(lse, lse_c)
    assert torch.equal(dqkv.view(torch.int16), d_c.view(torch.int16))


@pytest.mark.parametrize("D", [64, 128])
def test_one_token_segments_give_v_and_do(D):
    S = 200
    qkv, (q, k, v) = _qkv(1, S, 2, D, seed=5)
    seg_ids = torch.arange(S)[None]
    out, lse, dout, dqkv = _run(qkv, seg_ids, D, seed=5)
    assert torch.equal(out.view(torch.int16), v.contiguous().view(torch.int16))
    assert torch.equal(dqkv[:, :, :, 2].contiguous().view(torch.int16), dout.view(torch.int16))


@pytest.mark.parametrize("D", [64, 128])
def test_tiles_outside_the_segments_are_never_loaded(D):
    """A row split 256 | 768. NaN in the first segment's K and V: the second segment is finite and correct. NaN in the second
    segment's Q and dO: the first segment's gradients are finite and correct."""
    S, scale = 1024, 1.0 / math.sqrt(D)
    seg_ids = _rows_from_lengths([[256, 768]], S)
    st, en = ops.segment_bounds(seg_ids.to(DEV))
    clean, _ = _qkv(1, S, 2, D, seed=11)
    g = torch.Generator().manual_seed(12)
    dout = torch.randn(1, S, 2, D, generator=g).to(torch.bfloat16).to(DEV)

    def run(qkv, do):
        q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
        out, lse = ops.sdpa_segments_fwd(q, k, v, scale, st, en)
        d = torch.full_like(qkv, float("nan"))
        ops.sdpa_segments_bwd(q, k, v, out, do, lse, scale, st, en, d[:, :, :, 0], d[:, :, :, 1], d[:, :, :, 2])
        torch.cuda.synchronize()
        return out, lse, d

    # (a) poison the first segment's keys and values
    bad = clean.clone()
    bad[:, :256, :, 1:] = float("nan")
    out, lse, d = run(bad, dout)
    for t in (out[:, 256:], lse[:, :, 256:], d[:, 256:]):
        assert torch.isfinite(t.float()).all()
    _verify(clean, seg_ids, out, lse, dout, d, D, only=lambda b, s, e: s == 256)
    # (b) poison the second segment's queries and output gradients
    bad = clean.clone()
    bad[:, 256:, :, 0] = float("nan")
    bad_do = dout.clone()
    bad_do[:, 256:] = float("nan")
    out, lse, d = run(bad, bad_do)
    for t in (out[:, :256], lse[:, :, :256], d[:, :256]):
        assert torch.isfinite(t.float()).all()
    _verify(clean, seg_ids, out, lse, bad_do, d, D, only=lambda b, s, e: s == 0)


def test_second_run_is_bit_identical():
    S, D = 1024, 128
    seg_ids = _rows_from_lengths([_random_lengths(S, seed=1), [300, 700]], S)
    qkv, _ = _qkv(2, S, 2, D, seed=9)
    a = _run(qkv, seg_ids, D, seed=9)
    b = _run(qkv, seg_ids, D, seed=9)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))


def test_refusals():
    st, en = ops.segment_bounds(torch.zeros((1, 128), dtype=torch.int64, device=DEV))
    qkv = torch.zeros(1, 128, 2, 3, 96, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="head_dim 96"):
        ops.sdpa_segments_fwd(qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2], 0.1, st, en)
    q = torch.zeros(1, 128, 2, 64, dtype=torch.bfloat16, device=DEV)
    kv = torch.zeros(1, 256, 2, 64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="seq_q == seq_kv"):
        ops.sdpa_segments_fwd(q, kv, kv, 0.1, st, en)
    with pytest.raises(RuntimeError, match="seq_q == seq_kv"):
        ops.sdpa_segments_bwd(q, kv, kv, q, q, torch.zeros(1, 2, 128, device=DEV), 0.1, st, en, q.clone(), kv.clone(),
                              kv.clone())
