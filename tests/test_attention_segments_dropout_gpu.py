"""GPU: segment-masked causal attention with dropout on its probabilities (the causal segment form of
fsb_sdpa_{fwd,bwd} with p > 0, ops.sdpa_segments_*(drop=...)), the attention of packed GPT-2 training.

The keep mask of an element is that of the attention layout in include/fsb200.h at its row-relative (q, k), rebuilt here by
the numpy Philox of tests/philox_ref.py, never read from the library; the fp64 reference applies it under the block-diagonal
causal pattern of the row's segments. Exact answers: one segment per row is the causal dropout kernel bit for bit; one-token
segments give O = V Z / (1 - p) and dV = dO Z / (1 - p); p == 0 is the segment kernel without dropout. NaN planted in one
segment never reaches another."""
import math

import pytest
import torch

import philox_ref as R

from fsb200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
SEED, BASE, SITE = 0x2468_ACE0_1357_9BDF, (1 << 32) + 3, 4   # the stream base + site carries into the high word


def _base(v=BASE):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


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


def _case(B, S, D, seed, H=2):
    """q / k / v as strided views of the GPT-2 packed c_attn output [B, S, 3, heads, head_dim], and dO."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, S, 3, H, D, generator=g).to(torch.bfloat16).to(DEV)
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(DEV)
    return qkv, dout


def _run(qkv, dout, seg_ids, drop):
    D = qkv.shape[-1]
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    scale = 1.0 / math.sqrt(D)
    st, en = ops.segment_bounds(seg_ids.to(DEV))
    out, lse = ops.sdpa_segments_fwd(q, k, v, scale, st, en, drop=drop)
    dqkv = torch.full_like(qkv, float("nan"))
    ops.sdpa_segments_bwd(q, k, v, out, dout, lse, scale, st, en, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], drop=drop)
    torch.cuda.synchronize()
    return out, lse, dqkv


def _visible(seg_ids):
    """bool [B, 1, S, S]: key k visible to query q (same segment, k <= q)."""
    s = seg_ids.to(DEV)
    S = s.shape[1]
    # a segment is a maximal run: equal ids in two runs are still different segments
    run = torch.cumsum(torch.cat([torch.ones_like(s[:, :1]), (s[:, 1:] != s[:, :-1]).long()], 1), 1)
    same = run[:, :, None] == run[:, None, :]
    return (same & torch.ones(S, S, dtype=torch.bool, device=DEV).tril())[:, None]


def _check_fp64(qkv, dout, seg_ids, p, out, lse, dqkv, rows=None):
    """fp64 O, LSE, dQ, dK, dV under the block-diagonal causal pattern with the Philox keep mask; `rows` limits the check
    to some query / key positions (a bool [B, S] selection), for the NaN-isolation test."""
    B, S, _, H, D = qkv.shape
    scale = 1.0 / math.sqrt(D)
    keep = torch.from_numpy(R.attn_keep(SEED, BASE + SITE, B, H, S, S, p)).to(DEV, torch.float64)
    qf, kf, vf = (qkv[:, :, i].double().detach().requires_grad_(True) for i in range(3))
    vis = _visible(seg_ids)
    s = (torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale).masked_fill(~vis, float("-inf"))
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1) * keep / (1.0 - p), vf)
    sel = torch.ones(B, S, dtype=torch.bool, device=DEV) if rows is None else rows.to(DEV)
    o_err = (out.double() - ref).abs()[sel]
    assert not torch.isnan(o_err).any()
    assert o_err.max().item() < 2e-2 * max(1.0, ref.abs().max().item() / 4)
    l_err = (lse.double() * math.log(2.0) - torch.logsumexp(s, -1)).abs().permute(0, 2, 1)[sel]
    assert l_err.max().item() < 2e-3
    ref.backward(dout.double().masked_fill(~sel[:, :, None, None], 0.0))
    for name, got, want in (("dq", dqkv[:, :, 0], qf.grad), ("dk", dqkv[:, :, 1], kf.grad), ("dv", dqkv[:, :, 2], vf.grad)):
        g = got.double()[sel]
        assert not torch.isnan(g).any(), name
        err = (g - want[sel]).abs().max().item()
        assert err < 3e-2 * max(1.0, want.abs().max().item()), f"{name}: {err}"


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("S", [128, 200, 1024])
def test_segments_dropout_vs_fp64(S, p):
    """Seeded random lengths with one-token segments and a trailing pad segment in row 0; row 1 three segments."""
    seg_ids = _rows_from_lengths([_random_lengths(S, seed=S), [S // 2, S - S // 2 - 5, 5]], S)
    qkv, dout = _case(2, S, 64, seed=S)
    out, lse, dqkv = _run(qkv, dout, seg_ids, ops.Dropout(p, SEED, _base(), SITE))
    _check_fp64(qkv, dout, seg_ids, p, out, lse, dqkv)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_segments_dropout_at_tile_boundaries(p):
    """Segment edges at 63 / 64 / 65 and 127 / 128 / 129 (the 64-row streamed tiles and 128-row resident tiles)."""
    S = 1024
    layouts = [[63, 1, 65, 127, 1, 129, 128, 64], [64, 64, 129, 127, 128, 65, 63], [128, 128, 256, 512]]
    seg_ids = _rows_from_lengths(layouts, S)
    qkv, dout = _case(3, S, 64, seed=7)
    out, lse, dqkv = _run(qkv, dout, seg_ids, ops.Dropout(p, SEED, _base(), SITE))
    _check_fp64(qkv, dout, seg_ids, p, out, lse, dqkv)


@pytest.mark.parametrize("S", [256, 200])
def test_one_segment_is_the_causal_dropout_kernel_bit_for_bit(S):
    qkv, dout = _case(2, S, 64, seed=3)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    drop = ops.Dropout(0.1, SEED, _base(), SITE)
    out, lse, dqkv = _run(qkv, dout, torch.zeros((2, S), dtype=torch.int64), drop)
    o_c, lse_c = ops.sdpa_fwd(q, k, v, 0.125, True, drop=drop)
    d_c = torch.empty_like(qkv)
    ops.sdpa_bwd(q, k, v, o_c, dout, lse_c, 0.125, True, d_c[:, :, 0], d_c[:, :, 1], d_c[:, :, 2], drop=drop)
    torch.cuda.synchronize()
    assert torch.equal(out, o_c) and torch.equal(lse, lse_c)
    assert torch.equal(dqkv.view(torch.int16), d_c.view(torch.int16))


def test_one_token_segments_give_dropped_v_and_do():
    """Each query sees only itself: P = 1, so O = V Z / (1 - p) and dV = dO Z / (1 - p), Z the diagonal keep bit."""
    S, p = 200, 0.5
    qkv, dout = _case(1, S, 64, seed=5)
    out, lse, dqkv = _run(qkv, dout, torch.arange(S)[None], ops.Dropout(p, SEED, _base(), SITE))
    z = torch.from_numpy(R.attn_keep(SEED, BASE + SITE, 1, 2, S, S, p)).diagonal(dim1=2, dim2=3)   # [1, H, S]
    z = z.permute(0, 2, 1)[..., None].to(DEV)                                                        # [1, S, H, 1]
    assert 0 < int(z.sum()) < z.numel()
    scale = torch.tensor(2.0, dtype=torch.float32)   # 1 / (1 - 0.5): an exact power of two, so the products are exact
    want_o = torch.where(z, qkv[:, :, 2].float() * scale, 0.0).to(torch.bfloat16)
    want_dv = torch.where(z, dout.float() * scale, 0.0).to(torch.bfloat16)
    assert torch.equal(out, want_o)
    assert torch.equal(dqkv[:, :, 2], want_dv)


def test_nan_in_one_segment_never_reaches_another():
    """A row split 256 | 768. NaN in the first segment's q / k / v / dO: the second segment is finite and correct; NaN in the
    second one's: the first segment is."""
    S, p = 1024, 0.1
    seg_ids = _rows_from_lengths([[256, 768]], S)
    clean, dout = _case(1, S, 64, seed=11)
    drop = ops.Dropout(p, SEED, _base(), SITE)
    for lo, hi, other in ((0, 256, slice(256, S)), (256, S, slice(0, 256))):
        bad, bad_do = clean.clone(), dout.clone()
        bad[:, lo:hi] = float("nan")
        bad_do[:, lo:hi] = float("nan")
        out, lse, dqkv = _run(bad, bad_do, seg_ids, drop)
        for t in (out[:, other], lse[:, :, other], dqkv[:, other]):
            assert torch.isfinite(t.float()).all()
        rows = torch.zeros(1, S, dtype=torch.bool)
        rows[:, other] = True
        _check_fp64(clean, dout, seg_ids, p, out, lse, dqkv, rows=rows)


def test_second_run_is_bit_identical():
    S = 1024
    seg_ids = _rows_from_lengths([_random_lengths(S, seed=1), [300, 700]], S)
    qkv, dout = _case(2, S, 64, seed=9)
    drop = ops.Dropout(0.1, SEED, _base(), SITE)
    a, b = _run(qkv, dout, seg_ids, drop), _run(qkv, dout, seg_ids, drop)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))


def test_p_zero_is_the_segment_kernel_bit_for_bit():
    S = 1024
    seg_ids = _rows_from_lengths([_random_lengths(S, seed=2), [500, 524]], S)
    qkv, dout = _case(2, S, 64, seed=13)
    a = _run(qkv, dout, seg_ids, None)
    b = _run(qkv, dout, seg_ids, ops.Dropout(0.0, SEED, _base(), SITE))
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_form_refusals():
    drop = ops.Dropout(0.1, SEED, _base(), SITE)
    st, en = ops.segment_bounds(torch.zeros((1, 128), dtype=torch.int64, device=DEV))
    qkv = torch.zeros(1, 128, 3, 2, 128, dtype=torch.bfloat16, device=DEV)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    with pytest.raises(RuntimeError, match="head_dim 128 unsupported with p > 0"):
        ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, drop=drop)
    with pytest.raises(RuntimeError, match="head_dim 128 unsupported with p > 0"):
        ops.sdpa_segments_bwd(q, k, v, q, q, torch.zeros(1, 2, 128, device=DEV), 0.1, st, en, q.clone(), k.clone(),
                              v.clone(), drop=drop)
    ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, drop=ops.Dropout(0.0, SEED, _base(), SITE))   # p == 0: D 128 runs
    from fsb200 import lib as L
    qkv = torch.zeros(1, 128, 3, 2, 64, dtype=torch.bfloat16, device=DEV)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    o = torch.empty(1, 128, 2, 64, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(1, 2, 128, dtype=torch.float32, device=DEV)
    rs, hs = qkv.stride(1), qkv.stride(3)

    mask = torch.ones(1, 128, dtype=torch.uint8, device=DEV)

    def fwd(p, S=128, bounds=(st, en), kv_mask=None):
        L.call("fsb_sdpa_fwd", q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
               1, S, S, 2, 64, rs, rs, rs, o.stride(1), hs, hs, hs, o.stride(2), 0.125, 1, ops._p(kv_mask), None,
               *map(ops._p, bounds), None, None, p, SEED, _base().data_ptr(), SITE, None)
    for bad in (1.0, -0.1):
        with pytest.raises(RuntimeError, match="outside"):
            fwd(bad)
    with pytest.raises(RuntimeError, match="65536"):
        fwd(0.1, S=65537)
    for half in ((st, None), (None, en)):
        with pytest.raises(RuntimeError, match="null segment bounds"):
            fwd(0.1, bounds=half)
    with pytest.raises(RuntimeError, match="kv_mask"):
        fwd(0.1, kv_mask=mask)
    dq = torch.empty_like(o)

    def bwd(p, S=128, bounds=(st, en), kv_mask=None):
        delta = torch.empty(1, 2, 128, dtype=torch.float32, device=DEV)
        L.call("fsb_sdpa_bwd", q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), o.data_ptr(),
               lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), dq.data_ptr(), dq.data_ptr(), 1, S, S, 2, 64,
               rs, rs, rs, o.stride(1), o.stride(1), o.stride(1), o.stride(1), o.stride(1), hs, hs, hs, o.stride(2),
               o.stride(2), o.stride(2), o.stride(2), o.stride(2), 0.125, 1, ops._p(kv_mask), None, None, None, 0,
               *map(ops._p, bounds), None, None, p, SEED, _base().data_ptr(), SITE, None)
    with pytest.raises(RuntimeError, match="outside"):
        bwd(1.5)
    with pytest.raises(RuntimeError, match="65536"):
        bwd(0.1, S=65537)
    for half in ((st, None), (None, en)):
        with pytest.raises(RuntimeError, match="null segment bounds"):
            bwd(0.1, bounds=half)
    with pytest.raises(RuntimeError, match="kv_mask"):
        bwd(0.1, kv_mask=mask)
