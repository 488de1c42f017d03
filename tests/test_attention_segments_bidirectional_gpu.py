"""GPU: segment-masked bidirectional attention, with and without dropout on its probabilities
(fsb_sdpa_{fwd,bwd}_segments_bidirectional, ops.sdpa_segments_*(causal=False)), the attention of packed BERT / MegatronBERT
pretraining.

Key k is visible to query q iff both lie in the same segment. The keep mask of an element is that of the attention layout in
include/fsb200.h at its row-relative (q, k), rebuilt here by the numpy Philox of tests/philox_ref.py; the fp64 reference
applies it under the block-diagonal pattern of the row's segments. Exact answers: one segment per row is the non-causal
kernel without a key mask (p 0) and the non-causal dropout kernel (p > 0) bit for bit; one-token segments give
O = V Z / (1 - p) and dV = dO Z / (1 - p); p == 0 through the new pair is its dropout-free instantiation. NaN planted in one
segment never reaches another."""
import math

import pytest
import torch

import philox_ref as R

from fsb200 import lib as L
from fsb200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
SEED, BASE, SITE = 0x1357_9BDF_2468_ACE0, (1 << 32) + 5, 7


def _base(v=BASE):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _drop(p):
    return None if p == 0 else ops.Dropout(p, SEED, _base(), SITE)


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


def _case(B, S, seed, H=2, D=64):
    """q / k / v as strided views of a fused QKV projection output [B, S, 3, heads, head_dim], and dO."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, S, 3, H, D, generator=g).to(torch.bfloat16).to(DEV)
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(DEV)
    return qkv, dout


def _run(qkv, dout, seg_ids, drop):
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    scale = 1.0 / math.sqrt(qkv.shape[-1])
    st, en = ops.segment_bounds(seg_ids.to(DEV))
    out, lse = ops.sdpa_segments_fwd(q, k, v, scale, st, en, drop=drop, causal=False)
    dqkv = torch.full_like(qkv, float("nan"))
    ops.sdpa_segments_bwd(q, k, v, out, dout, lse, scale, st, en, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], drop=drop,
                          causal=False)
    torch.cuda.synchronize()
    return out, lse, dqkv


def _visible(seg_ids):
    """bool [B, 1, S, S]: key k visible to query q (same segment, either side)."""
    s = seg_ids.to(DEV)
    run = torch.cumsum(torch.cat([torch.ones_like(s[:, :1]), (s[:, 1:] != s[:, :-1]).long()], 1), 1)
    return (run[:, :, None] == run[:, None, :])[:, None]


def _check_fp64(qkv, dout, seg_ids, p, out, lse, dqkv, rows=None):
    """fp64 O, LSE, dQ, dK, dV under the block-diagonal pattern with the Philox keep mask; `rows` limits the check to some
    positions (a bool [B, S] selection), for the NaN-isolation test."""
    B, S, _, H, D = qkv.shape
    scale = 1.0 / math.sqrt(D)
    keep = torch.from_numpy(R.attn_keep(SEED, BASE + SITE, B, H, S, S, p)).to(DEV, torch.float64) if p > 0 else 1.0
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


LAYOUTS = {
    128: [[63, 1, 64], [64, 64], [1, 1, 1, 61, 64], [128], [127, 1], [100]],
    512: [[63, 1, 65, 127, 1, 128, 127], [64, 64, 128, 128, 128], [128, 256, 128], [512], [1] * 40 + [300, 100],
          [511, 1], [300]],
}


@pytest.mark.parametrize("p", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("S", [128, 512])
def test_bidirectional_segments_vs_fp64(S, p):
    """Segments ending at 63 / 64 / 127 / 128 (the 64-row streamed and 128-row resident tiles), one-token segments, a whole-row
    segment, a row ending in a pad segment."""
    seg_ids = _rows_from_lengths(LAYOUTS[S], S)
    qkv, dout = _case(seg_ids.shape[0], S, seed=S + int(10 * p))
    out, lse, dqkv = _run(qkv, dout, seg_ids, _drop(p))
    _check_fp64(qkv, dout, seg_ids, p, out, lse, dqkv)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("S", [256, 200])
def test_one_segment_is_the_non_causal_kernel_bit_for_bit(S, p):
    qkv, dout = _case(2, S, seed=3)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    drop = _drop(p)
    out, lse, dqkv = _run(qkv, dout, torch.zeros((2, S), dtype=torch.int64), drop)
    o_c, lse_c = ops.sdpa_fwd(q, k, v, 0.125, False, drop=drop)
    d_c = torch.empty_like(qkv)
    ops.sdpa_bwd(q, k, v, o_c, dout, lse_c, 0.125, False, d_c[:, :, 0], d_c[:, :, 1], d_c[:, :, 2], drop=drop)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), o_c.view(torch.int16)) and torch.equal(lse.view(torch.int32),
                                                                                       lse_c.view(torch.int32))
    assert torch.equal(dqkv.view(torch.int16), d_c.view(torch.int16))


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_one_token_segments_give_v_and_do(p):
    """Each query sees only itself: P = 1, so O = V Z / (1 - p) and dV = dO Z / (1 - p), Z the diagonal keep bit."""
    S = 200
    qkv, dout = _case(1, S, seed=5)
    out, lse, dqkv = _run(qkv, dout, torch.arange(S)[None], _drop(p))
    if p == 0:
        assert torch.equal(out, qkv[:, :, 2]) and torch.equal(dqkv[:, :, 2], dout)
        return
    z = torch.from_numpy(R.attn_keep(SEED, BASE + SITE, 1, 2, S, S, p)).diagonal(dim1=2, dim2=3)   # [1, H, S]
    z = z.permute(0, 2, 1)[..., None].to(DEV)                                                        # [1, S, H, 1]
    assert 0 < int(z.sum()) < z.numel()
    scale = torch.tensor(2.0, dtype=torch.float32)   # 1 / (1 - 0.5): an exact power of two, so the products are exact
    assert torch.equal(out, torch.where(z, qkv[:, :, 2].float() * scale, 0.0).to(torch.bfloat16))
    assert torch.equal(dqkv[:, :, 2], torch.where(z, dout.float() * scale, 0.0).to(torch.bfloat16))


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_nan_in_one_segment_never_reaches_another(p):
    """A row split 128 | 384. NaN in one segment's q / k / v / dO: the other segment is finite and correct, so the tiles
    of the other segment are never loaded. (Inside a tile two segments share, a masked P = 0 still multiplies the other
    segment's V or dO rows, and 0 * NaN is NaN, as for the key-padding mask.)"""
    S = 512
    seg_ids = _rows_from_lengths([[128, 384]], S)
    clean, dout = _case(1, S, seed=11)
    for lo, hi, other in ((0, 128, slice(128, S)), (128, S, slice(0, 128))):
        bad, bad_do = clean.clone(), dout.clone()
        bad[:, lo:hi] = float("nan")
        bad_do[:, lo:hi] = float("nan")
        out, lse, dqkv = _run(bad, bad_do, seg_ids, _drop(p))
        for t in (out[:, other], lse[:, :, other], dqkv[:, other]):
            assert torch.isfinite(t.float()).all()
        rows = torch.zeros(1, S, dtype=torch.bool)
        rows[:, other] = True
        _check_fp64(clean, dout, seg_ids, p, out, lse, dqkv, rows=rows)


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_second_run_is_bit_identical(p):
    S = 512
    seg_ids = _rows_from_lengths(LAYOUTS[512][:3], S)
    qkv, dout = _case(3, S, seed=9)
    a, b = _run(qkv, dout, seg_ids, _drop(p)), _run(qkv, dout, seg_ids, _drop(p))
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))


def test_p_zero_is_the_dropout_free_kernel_bit_for_bit():
    """Dropout(0.0) through the new pair runs the kernels drop=None runs (which passes no stream counter at all)."""
    S = 512
    seg_ids = _rows_from_lengths(LAYOUTS[512][:2], S)
    qkv, dout = _case(2, S, seed=13)
    a = _run(qkv, dout, seg_ids, None)
    b = _run(qkv, dout, seg_ids, ops.Dropout(0.0, SEED, _base(), SITE))
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_default_causal_keeps_the_causal_segment_kernels():
    """causal=True (the default) still launches fsb_sdpa_*_segments[_dropout]: the result is causal inside a segment."""
    S = 128
    seg_ids = _rows_from_lengths([[64, 64]], S)
    qkv, dout = _case(1, S, seed=17)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    st, en = ops.segment_bounds(seg_ids.to(DEV))
    o_def, _ = ops.sdpa_segments_fwd(q, k, v, 0.125, st, en)
    o_bi, _ = ops.sdpa_segments_fwd(q, k, v, 0.125, st, en, causal=False)
    torch.cuda.synchronize()
    assert torch.equal(o_def[:, 0], v[:, 0])              # the first query of a causal segment sees itself only
    assert not torch.equal(o_bi[:, 0], v[:, 0])


def test_refusals():
    st, en = ops.segment_bounds(torch.zeros((1, 128), dtype=torch.int64, device=DEV))
    qkv = torch.zeros(1, 128, 3, 2, 128, dtype=torch.bfloat16, device=DEV)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    with pytest.raises(RuntimeError, match="head_dim 128 unsupported"):
        ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, causal=False)
    with pytest.raises(RuntimeError, match="head_dim 128 unsupported"):
        ops.sdpa_segments_bwd(q, k, v, q, q, torch.zeros(1, 2, 128, device=DEV), 0.1, st, en, q.clone(), k.clone(),
                              v.clone(), causal=False)
    qkv = torch.zeros(1, 128, 3, 2, 64, dtype=torch.bfloat16, device=DEV)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    o = torch.empty(1, 128, 2, 64, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(1, 2, 128, dtype=torch.float32, device=DEV)
    rs, hs = qkv.stride(1), qkv.stride(3)

    def fwd(p, S=128, Skv=None, bounds=True):
        L.call("fsb_sdpa_fwd_segments_bidirectional", q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
               lse.data_ptr(), 1, S, S if Skv is None else Skv, 2, 64, rs, rs, rs, o.stride(1), hs, hs, hs, o.stride(2),
               0.125, st.data_ptr() if bounds else None, en.data_ptr() if bounds else None, p, SEED, _base().data_ptr(),
               SITE, None)
    for bad in (1.0, -0.1):
        with pytest.raises(RuntimeError, match="outside"):
            fwd(bad)
    with pytest.raises(RuntimeError, match="65536"):
        fwd(0.1, S=65537)
    with pytest.raises(RuntimeError, match="null segment bounds"):
        fwd(0.1, bounds=False)
    with pytest.raises(RuntimeError, match="seq_q == seq_kv"):
        fwd(0.0, Skv=64)
    dq = torch.empty_like(o)

    def bwd(p, S=128, Skv=None, bounds=True):
        delta = torch.empty(1, 2, 128, dtype=torch.float32, device=DEV)
        L.call("fsb_sdpa_bwd_segments_bidirectional", q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
               o.data_ptr(), lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), dq.data_ptr(), dq.data_ptr(), 1, S,
               S if Skv is None else Skv, 2, 64, rs, rs, rs, o.stride(1), o.stride(1), o.stride(1), o.stride(1),
               o.stride(1), hs, hs, hs, o.stride(2), o.stride(2), o.stride(2), o.stride(2), o.stride(2), 0.125,
               st.data_ptr() if bounds else None, en.data_ptr() if bounds else None, p, SEED, _base().data_ptr(), SITE,
               None)
    with pytest.raises(RuntimeError, match="outside"):
        bwd(1.5)
    with pytest.raises(RuntimeError, match="65536"):
        bwd(0.1, S=65537)
    with pytest.raises(RuntimeError, match="null segment bounds"):
        bwd(0.1, bounds=False)
    with pytest.raises(RuntimeError, match="seq_q == seq_kv"):
        bwd(0.0, Skv=64)

