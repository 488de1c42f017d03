"""GPU: the packed attention of mT5 / Randeng-T5 fine-tuning, with and without dropout on its probabilities:
  * segment-masked self-attention with the relative-position bias (the biased segment form of fsb_sdpa_{fwd,bwd},
    ops.sdpa_segments_*(rel_bias=...)): bidirectional inside each segment (the encoder) or causal inside it (the decoder);
  * segment-paired cross-attention between rows of different lengths (the cross segment form of fsb_sdpa_{fwd,bwd},
    ops.sdpa_segments_*(kv_bounds=...)): decoder segment x of a row sees the encoder segment with id x of the same row.

The fp64 reference builds the scores with the bias vector gathered at k - q, masks them with the segment pattern and applies
the keep mask of the attention layout of include/fsb200.h at each element's row-relative (q, k) (tests/philox_ref.py); the
bias gradient is its autograd gradient. Exact answers: one segment per row is the unsegmented kernel bit for bit (the bias
gradient included); one-token segments with exactly representable inputs give O == V and add exactly 0 to the bias
gradient; p == 0 is the dropout-free kernel; queries without keys and keys without queries give exact zeros with every
output written; NaN planted in one segment never reaches another; a NaN-poisoned workspace still gives the fp64 bias
gradient (the reduction reads only the slots the dQ pass wrote)."""
import math

import pytest
import torch

import philox_ref as R

from fsb200 import lib as L
from fsb200 import ops
from fsb200.models.base import cross_segment_bounds

pytestmark = pytest.mark.gpu

DEV = "cuda"
SEED, BASE, SITE = 0x2468_ACE0_1357_9BDF, (1 << 32) + 9, 5
H, D = 2, 64


def _base(v=BASE):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _drop(p):
    return None if p == 0 else ops.Dropout(p, SEED, _base(), SITE)


def _ids(layouts, S):
    """segment ids [B, S] from per-row segment lengths; a short sum leaves a trailing segment (the pad tail) with the next id."""
    ids = torch.zeros((len(layouts), S), dtype=torch.int64)
    for b, lens in enumerate(layouts):
        t = 0
        for k, n in enumerate(lens):
            ids[b, t:t + n] = k
            t += n
        assert t <= S
        ids[b, t:] = len(lens)
    return ids


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _same(a, b):
    return all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ self-attention + bias
def _self_case(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, S, 3, H, D, generator=g).to(torch.bfloat16).to(DEV)
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(DEV)
    rel = (2.0 * torch.randn(H, 2 * S - 1, generator=g)).to(DEV)
    return qkv, dout, rel


def _run_bias(qkv, dout, rel, seg_ids, causal, drop, scale=0.125):
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    st, en = ops.segment_bounds(seg_ids.to(DEV))
    out, lse = ops.sdpa_segments_fwd(q, k, v, scale, st, en, drop=drop, causal=causal, rel_bias=rel)
    dqkv = torch.full_like(qkv, float("nan"))
    drel = torch.zeros_like(rel)
    ops.sdpa_segments_bwd(q, k, v, out, dout, lse, scale, st, en, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], drop=drop,
                          causal=causal, rel_bias=rel, drel_bias=drel)
    torch.cuda.synchronize()
    return out, lse, dqkv, drel


def _self_visible(seg_ids, causal):
    s = seg_ids.to(DEV)
    run = torch.cumsum(torch.cat([torch.ones_like(s[:, :1]), (s[:, 1:] != s[:, :-1]).long()], 1), 1)
    vis = run[:, :, None] == run[:, None, :]
    if causal:
        S = s.shape[1]
        vis = vis & torch.ones(S, S, dtype=torch.bool, device=DEV).tril()
    return vis[:, None]


def _fp64(q, k, v, dout, vis, p, rel=None, scale=0.125, sel_q=None):
    """fp64 O, LSE (natural log), dQ, dK, dV, dRel under `vis` [B, 1, Sq, Skv]. Queries without a visible key get O = 0 and
    no gradient. sel_q: bool [B, Sq] limiting the dO rows that enter the backward (NaN isolation)."""
    B, Sq = q.shape[:2]
    Skv = k.shape[1]
    keep = torch.from_numpy(R.attn_keep(SEED, BASE + SITE, B, H, Sq, Skv, p)).to(DEV, torch.float64) if p > 0 else 1.0
    qf, kf, vf = (t.double().detach().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    relf = None
    if rel is not None:
        relf = rel.double().detach().requires_grad_(True)
        idx = torch.arange(Skv, device=DEV)[None, :] - torch.arange(Sq, device=DEV)[:, None] + Sq - 1
        s = s + relf[:, idx][None]
    any_key = vis.any(-1, keepdim=True)
    s = s.masked_fill(~vis, float("-inf")).masked_fill(~any_key, 0.0)
    lse = torch.logsumexp(s, -1)
    prob = torch.softmax(s, -1) * any_key
    o = torch.einsum("bhqk,bkhd->bqhd", prob * keep / (1.0 - p), vf)
    g = dout.double()
    if sel_q is not None:
        g = g.masked_fill(~sel_q.to(DEV)[:, :, None, None], 0.0)
    o.backward(g)
    return o.detach(), lse.detach(), any_key[:, 0, :, 0], qf.grad, kf.grad, vf.grad, None if relf is None else relf.grad


def _close(name, got, want, tol):
    got = got.double()
    assert not torch.isnan(got).any(), name
    err = (got - want).abs().max().item()
    assert err < tol * max(1.0, want.abs().max().item()), f"{name}: {err}"


def _check_self(qkv, dout, rel, seg_ids, causal, p, res, sel=None, scale=0.125):
    out, lse, dqkv, drel = res
    vis = _self_visible(seg_ids, causal)
    o, l_ref, _, dq, dk, dv, dr = _fp64(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], dout, vis, p, rel, scale, sel)
    m = torch.ones(qkv.shape[:2], dtype=torch.bool, device=DEV) if sel is None else sel.to(DEV)
    _close("o", out[m], o[m], 2e-2)
    _close("lse", (lse.double() * math.log(2.0)).permute(0, 2, 1)[m], l_ref.permute(0, 2, 1)[m], 2e-3)
    for name, got, want in (("dq", dqkv[:, :, 0], dq), ("dk", dqkv[:, :, 1], dk), ("dv", dqkv[:, :, 2], dv)):
        _close(name, got[m], want[m], 3e-2)
    if sel is None:
        _close("drel", drel, dr, 2e-2)


LAYOUTS = {
    128: [[63, 1, 64], [64, 64], [1, 1, 1, 61, 64], [128], [127, 1], [100]],
    200: [[63, 1, 65, 71], [128, 72], [1] * 10 + [150], [199]],
    512: [[63, 1, 65, 127, 1, 128, 127], [64, 64, 128, 128, 128], [128, 256, 128], [512], [1] * 40 + [300, 100],
          [511, 1], [300]],
}


@pytest.mark.parametrize("p", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("S", [128, 200, 512])
def test_bias_segments_vs_fp64(S, causal, p):
    """Segments ending on and off the 64-row streamed and 128-row resident tiles, one-token segments, a whole-row segment,
    a row ending in a pad segment; O, LSE, dQ, dK, dV and the bias gradient."""
    seg_ids = _ids(LAYOUTS[S], S)
    qkv, dout, rel = _self_case(seg_ids.shape[0], S, seed=S + int(10 * p) + 100 * causal)
    _check_self(qkv, dout, rel, seg_ids, causal, p, _run_bias(qkv, dout, rel, seg_ids, causal, _drop(p)))


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("S", [256, 200])
def test_one_segment_is_the_bias_kernel_bit_for_bit(S, causal, p):
    """One segment per row: fsb_sdpa_{fwd,bwd}[_dropout] with the same bias and causal flag, bias gradient included."""
    qkv, dout, rel = _self_case(2, S, seed=3)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    drop = _drop(p)
    got = _run_bias(qkv, dout, rel, torch.zeros((2, S), dtype=torch.int64), causal, drop)
    o, lse = ops.sdpa_fwd(q, k, v, 0.125, causal, rel_bias=rel, drop=drop)
    d = torch.empty_like(qkv)
    drel = torch.zeros_like(rel)
    ops.sdpa_bwd(q, k, v, o, dout, lse, 0.125, causal, d[:, :, 0], d[:, :, 1], d[:, :, 2], rel_bias=rel, drel_bias=drel,
                 drop=drop)
    torch.cuda.synchronize()
    assert _same(got, (o, lse, d, drel))


@pytest.mark.parametrize("causal", [False, True])
def test_one_token_segments_give_v_and_no_bias_gradient(causal):
    """Each query sees only itself. With Q = 0 and biases that are powers of two (bias * log2(e) exact in fp32) P is exactly
    1, so O == V and dV == dO; with dO and V in {-1, 0, 1} the sums dP = dO . V and delta = dO . O are exact in any order,
    so every dS is exactly 0 and the bias gradient gains exactly nothing."""
    S = 200
    g = torch.Generator().manual_seed(5)
    qkv = torch.randn(1, S, 3, H, D, generator=g).to(torch.bfloat16)
    qkv[:, :, 0] = 0.0
    qkv[:, :, 2] = torch.randint(-1, 2, (1, S, H, D), generator=g).to(torch.bfloat16)
    dout = torch.randint(-1, 2, (1, S, H, D), generator=g).to(torch.bfloat16).to(DEV)
    rel = torch.ldexp(torch.ones(H, 2 * S - 1), torch.randint(-3, 3, (H, 2 * S - 1), generator=g)).to(DEV)
    qkv = qkv.to(DEV)
    out, lse, dqkv, drel = _run_bias(qkv, dout, rel, torch.arange(S)[None], causal, None)
    assert torch.equal(out, qkv[:, :, 2]) and torch.equal(dqkv[:, :, 2], dout)
    assert torch.equal(drel, torch.zeros_like(drel))


def test_poisoned_workspace_still_gives_the_fp64_bias_gradient():
    """The bias-gradient workspace is filled with NaN before the backward: the reduction reads only the per-step slots the
    dQ pass wrote (the steps the segment bounds skip are neither written nor read)."""
    S = 512
    seg_ids = _ids(LAYOUTS[512], S)
    B = seg_ids.shape[0]
    qkv, dout, rel = _self_case(B, S, seed=21)
    ws = ops.workspace(int(L.load().fsb_sdpa_bwd_workspace_bytes(B, S, S, H)), torch.device(DEV), "sdpa_dbias")
    for causal in (False, True):
        ws.view(torch.float32)[: ws.numel() // 4].fill_(float("nan"))
        res = _run_bias(qkv, dout, rel, seg_ids, causal, None)
        _check_self(qkv, dout, rel, seg_ids, causal, 0.0, res)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_bias_nan_in_one_segment_never_reaches_another(p, causal):
    """A row split 128 | 384 with NaN in one segment's q / k / v / dO: the other segment's outputs are finite and correct.
    (The bias gradient sums over every segment, so it is not checked here.)"""
    S = 512
    seg_ids = _ids([[128, 384]], S)
    clean, dout, rel = _self_case(1, S, seed=11)
    for lo, hi, other in ((0, 128, slice(128, S)), (128, S, slice(0, 128))):
        bad, bad_do = clean.clone(), dout.clone()
        bad[:, lo:hi] = float("nan")
        bad_do[:, lo:hi] = float("nan")
        res = _run_bias(bad, bad_do, rel, seg_ids, causal, _drop(p))
        for t in (res[0][:, other], res[1][:, :, other], res[2][:, other]):
            assert torch.isfinite(t.float()).all()
        rows = torch.zeros(1, S, dtype=torch.bool)
        rows[:, other] = True
        _check_self(clean, dout, rel, seg_ids, causal, p, res, sel=rows)


# ------------------------------------------------------------------------------------------------ cross-attention
def _cross_case(B, Sd, Se, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Sd, H, D, generator=g).to(torch.bfloat16).to(DEV)
    kv = torch.randn(B, Se, 2, H, D, generator=g).to(torch.bfloat16).to(DEV)
    dout = torch.randn(B, Sd, H, D, generator=g).to(torch.bfloat16).to(DEV)
    return q, kv, dout


def _run_cross(q, kv, dout, dec_ids, enc_ids, drop, scale=0.125):
    kvb, qb = cross_segment_bounds(dec_ids.to(DEV), enc_ids.to(DEV))
    k, v = kv[:, :, 0], kv[:, :, 1]
    out = torch.full_like(q, float("nan"))
    out, lse = ops.sdpa_segments_fwd(q, k, v, scale, *kvb, out=out, drop=drop, causal=False, kv_bounds=qb)
    dq = torch.full_like(q, float("nan"))
    dkv = torch.full_like(kv, float("nan"))
    ops.sdpa_segments_bwd(q, k, v, out, dout, lse, scale, *kvb, dq, dkv[:, :, 0], dkv[:, :, 1], drop=drop, causal=False,
                          kv_bounds=qb)
    torch.cuda.synchronize()
    return out, lse, dq, dkv


def _check_cross(q, kv, dout, dec_ids, enc_ids, p, res, sel=None):
    out, lse, dq, dkv = res
    vis = (dec_ids.to(DEV)[:, :, None] == enc_ids.to(DEV)[:, None, :])[:, None]
    o, l_ref, has, dq_r, dk_r, dv_r, _ = _fp64(q, kv[:, :, 0], kv[:, :, 1], dout, vis, p, sel_q=sel)
    m = torch.ones(q.shape[:2], dtype=torch.bool, device=DEV) if sel is None else sel.to(DEV)
    _close("o", out[m], o[m], 2e-2)
    lm = m & has
    _close("lse", (lse.double() * math.log(2.0)).permute(0, 2, 1)[lm], l_ref.permute(0, 2, 1)[lm], 2e-3)
    _close("dq", dq[m], dq_r[m], 3e-2)
    if sel is None:
        _close("dk", dkv[:, :, 0], dk_r, 3e-2)
        _close("dv", dkv[:, :, 1], dv_r, 3e-2)


# (decoder segment lengths per row, encoder segment lengths per row); a short sum leaves a pad tail with the next id, which
# pairs with the other side's tail when both have one and is an empty range when only one does
CROSS = {
    (512, 114): ([[63, 1, 65, 127, 1, 128, 127], [64, 64, 128, 128], [500], [512], [1] * 40 + [300]],
                 [[10, 20, 5, 30, 1, 20, 28], [30, 30, 27, 27], [114], [100], [1] * 40 + [74]]),
    (200, 77): ([[63, 1, 65, 71], [128, 72], [1] * 10 + [150], [199], [64]],
                [[20, 7, 30, 20], [40, 37], [7] * 11, [77], [77]]),
    (128, 256): ([[63, 1, 64], [64, 64], [100]],
                 [[127, 1, 128], [64, 64], [256]]),
}


@pytest.mark.parametrize("p", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("shape", list(CROSS))
def test_cross_segments_vs_fp64(shape, p):
    Sd, Se = shape
    dl, el = CROSS[shape]
    dec_ids, enc_ids = _ids(dl, Sd), _ids(el, Se)
    q, kv, dout = _cross_case(len(dl), Sd, Se, seed=Sd + Se + int(10 * p))
    _check_cross(q, kv, dout, dec_ids, enc_ids, p, _run_cross(q, kv, dout, dec_ids, enc_ids, _drop(p)))


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("shape", [(512, 114), (200, 77), (128, 256)])
def test_one_cross_segment_is_the_unmasked_kernel_bit_for_bit(shape, p):
    Sd, Se = shape
    q, kv, dout = _cross_case(2, Sd, Se, seed=7)
    drop = _drop(p)
    got = _run_cross(q, kv, dout, torch.zeros((2, Sd), dtype=torch.int64), torch.zeros((2, Se), dtype=torch.int64), drop)
    k, v = kv[:, :, 0], kv[:, :, 1]
    o, lse = ops.sdpa_fwd(q, k, v, 0.125, False, drop=drop)
    dq, dkv = torch.empty_like(q), torch.empty_like(kv)
    ops.sdpa_bwd(q, k, v, o, dout, lse, 0.125, False, dq, dkv[:, :, 0], dkv[:, :, 1], drop=drop)
    torch.cuda.synchronize()
    assert _same(got, (o, lse, dq, dkv))


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_empty_cross_ranges_give_exact_zeros(p):
    """Row 0: the decoder has a pad tail (id 2) and the encoder is full (ids 0, 1 only), so the tail's queries see no key:
    O = 0, LSE = +inf, dQ = 0. Row 1: the encoder has a pad tail (id 2) the full decoder never pairs with: its keys get
    dK = dV = 0. Row 2: whole tiles of either side without a partner. Outputs start as NaN, so every element is written."""
    Sd, Se = 200, 77
    dec_ids = _ids([[50, 30], [120, 80], [60]], Sd)          # row 2: decoder id 1 covers 60..199
    enc_ids = torch.stack([_ids([[40, 37]], Se)[0], _ids([[30, 20]], Se)[0], torch.full((Se,), 5)])
    q, kv, dout = _cross_case(3, Sd, Se, seed=13)
    out, lse, dq, dkv = _run_cross(q, kv, dout, dec_ids, enc_ids, _drop(p))
    lonely_q = torch.zeros(3, Sd, dtype=torch.bool)
    lonely_q[0, 80:], lonely_q[2, :] = True, True
    lonely_k = torch.zeros(3, Se, dtype=torch.bool)
    lonely_k[1, 50:], lonely_k[2, :] = True, True
    assert torch.equal(out[lonely_q], torch.zeros_like(out[lonely_q]))
    assert torch.equal(dq[lonely_q], torch.zeros_like(dq[lonely_q]))
    assert bool((lse.permute(0, 2, 1)[lonely_q] == float("inf")).all())
    assert torch.equal(dkv[lonely_k], torch.zeros_like(dkv[lonely_k]))
    _check_cross(q, kv, dout, dec_ids, enc_ids, p, (out, lse, dq, dkv))


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_cross_nan_in_one_segment_never_reaches_another(p):
    """Decoder 128 | 384, encoder 128 | 128: NaN in one pair's q / k / v / dO leaves the other pair finite and correct, so
    the other pair's tiles are never loaded. (Both splits sit on tile boundaries: inside a tile two pairs share, a masked
    P = 0 still multiplies the other pair's V or dO rows, and 0 * NaN is NaN, as for the key-padding mask.)"""
    Sd, Se = 512, 256
    dec_ids, enc_ids = _ids([[128, 384]], Sd), _ids([[128, 128]], Se)
    clean_q, clean_kv, dout = _cross_case(1, Sd, Se, seed=17)
    for (dlo, dhi), (elo, ehi), other in (((0, 128), (0, 128), slice(128, Sd)), ((128, Sd), (128, Se), slice(0, 128))):
        q, kv, do = clean_q.clone(), clean_kv.clone(), dout.clone()
        q[:, dlo:dhi] = float("nan")
        do[:, dlo:dhi] = float("nan")
        kv[:, elo:ehi] = float("nan")
        res = _run_cross(q, kv, do, dec_ids, enc_ids, _drop(p))
        other_k = slice(128, Se) if elo == 0 else slice(0, 128)
        for t in (res[0][:, other], res[1][:, :, other], res[2][:, other], res[3][:, other_k]):
            assert torch.isfinite(t.float()).all()
        rows = torch.zeros(1, Sd, dtype=torch.bool)
        rows[:, other] = True
        _check_cross(clean_q, clean_kv, dout, dec_ids, enc_ids, p, res, sel=rows)


# ------------------------------------------------------------------------------------------------ both forms
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_second_run_is_bit_identical(p):
    S = 512
    seg_ids = _ids(LAYOUTS[512][:3], S)
    qkv, dout, rel = _self_case(3, S, seed=9)
    for causal in (False, True):
        assert _same(_run_bias(qkv, dout, rel, seg_ids, causal, _drop(p)),
                     _run_bias(qkv, dout, rel, seg_ids, causal, _drop(p)))
    dl, el = CROSS[(512, 114)]
    dec_ids, enc_ids = _ids(dl, 512), _ids(el, 114)
    q, kv, do = _cross_case(len(dl), 512, 114, seed=9)
    assert _same(_run_cross(q, kv, do, dec_ids, enc_ids, _drop(p)), _run_cross(q, kv, do, dec_ids, enc_ids, _drop(p)))


def test_p_zero_is_the_dropout_free_kernel_bit_for_bit():
    """Dropout(0.0) runs the kernels drop=None runs (which reads no stream counter)."""
    S = 512
    seg_ids = _ids(LAYOUTS[512][:2], S)
    qkv, dout, rel = _self_case(2, S, seed=13)
    zero = ops.Dropout(0.0, SEED, _base(), SITE)
    for causal in (False, True):
        assert _same(_run_bias(qkv, dout, rel, seg_ids, causal, None), _run_bias(qkv, dout, rel, seg_ids, causal, zero))
    dl, el = CROSS[(200, 77)]
    dec_ids, enc_ids = _ids(dl, 200), _ids(el, 77)
    q, kv, do = _cross_case(len(dl), 200, 77, seed=13)
    assert _same(_run_cross(q, kv, do, dec_ids, enc_ids, None), _run_cross(q, kv, do, dec_ids, enc_ids, zero))


def _strides(*ts):
    return [t.stride(1) for t in ts], [t.stride(2) for t in ts]


def test_form_refusals():
    S = 128
    st, en = ops.segment_bounds(torch.zeros((1, S), dtype=torch.int64, device=DEV))
    rel = torch.zeros(H, 2 * S - 1, device=DEV)
    for d in (128, 64):
        qkv = torch.zeros(1, S, 3, H, d, dtype=torch.bfloat16, device=DEV)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        if d == 128:
            with pytest.raises(RuntimeError, match="head_dim 128 unsupported"):
                ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, causal=False, rel_bias=torch.zeros(H, 2 * S - 1, device=DEV))
            with pytest.raises(RuntimeError, match="head_dim 128 unsupported"):
                ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, causal=False, kv_bounds=(st, en))
    o = torch.empty(1, S, H, D, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(1, H, S, dtype=torch.float32, device=DEV)
    delta = torch.empty(1, H, S, dtype=torch.float32, device=DEV)
    rs, hs = qkv.stride(1), qkv.stride(3)
    ors, ohs = o.stride(1), o.stride(2)
    ws_need = int(L.load().fsb_sdpa_bwd_workspace_bytes(1, S, S, H))
    ws = torch.empty(ws_need, dtype=torch.uint8, device=DEV)

    def fwd(p, S=S, Skv=S, bounds=(st, en), qb=(None, None), causal=1, bias=True, d=64):
        L.call("fsb_sdpa_fwd", q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), 1, S, Skv, H, d,
               rs, rs, rs, ors, hs, hs, hs, ohs, 0.125, causal, None, rel.data_ptr() if bias else None,
               *map(ops._p, bounds + qb), p, SEED, _base().data_ptr(), SITE, None)

    def bwd(p, S=S, Skv=S, bounds=(st, en), qb=(None, None), causal=1, bias=True, drel=False, ws_bytes=ws_need):
        L.call("fsb_sdpa_bwd", q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), o.data_ptr(), lse.data_ptr(),
               delta.data_ptr(), o.data_ptr(), o.data_ptr(), o.data_ptr(), 1, S, Skv, H, 64, rs, rs, rs, ors, ors, ors,
               ors, ors, hs, hs, hs, ohs, ohs, ohs, ohs, ohs, 0.125, causal, None, rel.data_ptr() if bias else None,
               rel.data_ptr() if drel else None, ws.data_ptr(), ws_bytes, *map(ops._p, bounds + qb), p, SEED,
               _base().data_ptr(), SITE, None)

    biased, cross = dict(causal=1, bias=True), dict(causal=0, bias=False, qb=(st, en))
    for call in (fwd, bwd):
        for form in (biased, cross):
            for bad in (1.0, -0.1):
                with pytest.raises(RuntimeError, match="outside"):
                    call(bad, **form)
            with pytest.raises(RuntimeError, match="65536"):
                call(0.1, S=65537, Skv=65537, **form)
            for half in ((st, None), (None, en)):
                with pytest.raises(RuntimeError, match="null segment bounds"):
                    call(0.1, **dict(form, bounds=half))
        # the key-side bounds of the cross form: both or neither, and only beside the query-side ones
        for qb, bounds in (((st, None), (st, en)), ((None, en), (st, en)), ((st, en), (None, None))):
            with pytest.raises(RuntimeError, match="null segment bounds"):
                call(0.1, **dict(cross, qb=qb, bounds=bounds))
        with pytest.raises(RuntimeError, match="seq_q == seq_kv"):
            call(0.0, Skv=64, **biased)
        # the cross form has no causal mask and no bias
        for extra in (dict(causal=1), dict(bias=True)):
            with pytest.raises(RuntimeError, match="cross segments take no causal mask and no rel_bias"):
                call(0.0, **dict(cross, **extra))
    with pytest.raises(RuntimeError, match="workspace"):
        bwd(0.0, drel=True, ws_bytes=ws_need - 16, **biased)
    with pytest.raises(RuntimeError, match="head_dim 128 unsupported"):
        fwd(0.0, d=128, **cross)
    # ops-level: no bias with the cross form, the cross form is not causal, drel_bias needs rel_bias
    with pytest.raises(RuntimeError, match="takes no rel_bias"):
        ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, causal=False, rel_bias=rel, kv_bounds=(st, en))
    with pytest.raises(RuntimeError, match="no causal mask"):
        ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, kv_bounds=(st, en))
    with pytest.raises(RuntimeError, match="drel_bias needs rel_bias"):
        ops.sdpa_segments_bwd(q, k, v, o, o, lse, 0.1, st, en, o.clone(), o.clone(), o.clone(), drel_bias=rel)
