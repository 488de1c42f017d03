"""GPU: causal attention at head_dim 96 (the 3.5B Wenzhong / Yuyuan GPT-2: 32 heads x 96), in every form GPT-2 launches:
causal with an optional key mask, the same with dropout on the probabilities, and packed causal segments with and without
dropout (the dense and causal segment forms of fsb_sdpa_{fwd,bwd} at head_dim 96).

q / k / v are strided views of one packed [B, S, 3, H, 96] tensor, as GPT-2's c_attn output. References are fp64; the keep
masks are rebuilt by the numpy Philox of tests/philox_ref.py. The D = 96 kernels stage whole 64-column panels, as the
D = 128 kernels do, and contract S = Q K^T over 6 k16 steps: their forward is bit for bit the D = 128 forward on copies of
q, k, v zero-padded to 128 columns (the two extra k-steps of D = 128 add exact zeros)."""
import math

import pytest
import torch

import footprint as F
import philox_ref as R

from fsb200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"
D = 96
SEED, BASE, SITE = 0x1357_9BDF_2468_ACE0, (1 << 32) + 11, 6


def _base():
    return torch.tensor([BASE], dtype=torch.int64, device=DEV)


def _drop(p):
    return None if p is None else ops.Dropout(p, SEED, _base(), SITE)


def _case(B, S, H, seed, heads_total=None):
    """qkv [B, S, 3, heads_total, 96] bf16 and dO [B, S, H, 96]; the attention runs on heads [0, H)."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, S, 3, heads_total or H, D, generator=g).to(torch.bfloat16).to(DEV)
    dout = torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(DEV)
    return qkv, dout


def _key_mask(B, S):
    """Row 0 sees every key; row b > 0 has its last S // (3 b) keys masked (key 0 always visible)."""
    m = torch.ones(B, S, dtype=torch.uint8)
    for b in range(1, B):
        n = S // (3 * b)
        if 0 < n < S:
            m[b, S - n:] = 0
    return m.to(DEV)


def _seg_ids(layouts, S):
    ids = torch.zeros((len(layouts), S), dtype=torch.int64)
    for b, lens in enumerate(layouts):
        t = 0
        for k, n in enumerate(lens):
            ids[b, t:t + n] = k
            t += n
        ids[b, t:] = len(lens)
    return ids.to(DEV)


def _visible(B, S, mask=None, seg_ids=None):
    """bool [B, 1, S, S]: causal, under the key mask or inside each query's segment."""
    vis = torch.ones(S, S, dtype=torch.bool, device=DEV).tril()[None, None].expand(B, 1, S, S)
    if mask is not None:
        vis = vis & mask.bool()[:, None, None, :]
    if seg_ids is not None:
        s = seg_ids
        run = torch.cumsum(torch.cat([torch.ones_like(s[:, :1]), (s[:, 1:] != s[:, :-1]).long()], 1), 1)
        vis = vis & (run[:, :, None] == run[:, None, :])[:, None]
    return vis


def _run(qkv, dout, H, mask=None, seg_ids=None, p=None, dqkv=None):
    """Forward and backward over heads [0, H) of qkv; dq / dk / dv land in the matching views of dqkv (NaN-filled)."""
    q, k, v = (qkv[:, :, i, :H] for i in range(3))
    scale = 1.0 / math.sqrt(D)
    drop = _drop(p)
    dqkv = torch.full_like(qkv, float("nan")) if dqkv is None else dqkv
    dq, dk, dv = (dqkv[:, :, i, :H] for i in range(3))
    if seg_ids is None:
        out, lse = ops.sdpa_fwd(q, k, v, scale, True, kv_mask=mask, drop=drop)
        ops.sdpa_bwd(q, k, v, out, dout, lse, scale, True, dq, dk, dv, kv_mask=mask, drop=drop)
    else:
        st, en = ops.segment_bounds(seg_ids)
        out, lse = ops.sdpa_segments_fwd(q, k, v, scale, st, en, drop=drop)
        ops.sdpa_segments_bwd(q, k, v, out, dout, lse, scale, st, en, dq, dk, dv, drop=drop)
    torch.cuda.synchronize()
    return out, lse, dqkv


def _check_fp64(qkv, dout, H, out, lse, dqkv, mask=None, seg_ids=None, p=None):
    """Tolerances of tests/test_attention_segments_dropout_gpu.py (bf16 P and O against fp64)."""
    B, S = qkv.shape[:2]
    scale = 1.0 / math.sqrt(D)
    qf, kf, vf = (qkv[:, :, i, :H].double().detach().requires_grad_(True) for i in range(3))
    vis = _visible(B, S, mask, seg_ids)
    s = (torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale).masked_fill(~vis, float("-inf"))
    prob = torch.softmax(s, -1)
    if p:
        keep = torch.from_numpy(R.attn_keep(SEED, BASE + SITE, B, H, S, S, p)).to(DEV, torch.float64)
        prob = prob * keep / (1.0 - p)
    ref = torch.einsum("bhqk,bkhd->bqhd", prob, vf)
    err = (out.double() - ref).abs()
    assert not torch.isnan(err).any()
    assert err.max().item() < 2e-2 * max(1.0, ref.abs().max().item() / 4), err.max().item()
    l_err = (lse.double() * math.log(2.0) - torch.logsumexp(s, -1)).abs()
    assert l_err.max().item() < 2e-3, l_err.max().item()
    ref.backward(dout.double())
    for name, i, want in (("dq", 0, qf.grad), ("dk", 1, kf.grad), ("dv", 2, vf.grad)):
        got = dqkv[:, :, i, :H].double()
        assert not torch.isnan(got).any(), name
        e = (got - want).abs().max().item()
        assert e < 3e-2 * max(1.0, want.abs().max().item()), f"{name}: {e}"


# ------------------------------------------------------------------------------------------------ against fp64
@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "keymask"])
@pytest.mark.parametrize("S", [1, 63, 64, 65, 127, 129, 1000, 1024])
def test_causal_vs_fp64(S, masked):
    B, H = 2, 3
    qkv, dout = _case(B, S, H, seed=S)
    mask = _key_mask(B, S) if masked else None
    out, lse, dqkv = _run(qkv, dout, H, mask=mask)
    _check_fp64(qkv, dout, H, out, lse, dqkv, mask=mask)


@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "keymask"])
@pytest.mark.parametrize("S", [65, 129, 1024])
def test_causal_dropout_vs_fp64(S, masked):
    B, H = 2, 2
    qkv, dout = _case(B, S, H, seed=100 + S)
    mask = _key_mask(B, S) if masked else None
    out, lse, dqkv = _run(qkv, dout, H, mask=mask, p=0.1)
    _check_fp64(qkv, dout, H, out, lse, dqkv, mask=mask, p=0.1)


LAYOUTS = {
    1024: [[63, 1, 65, 127, 1, 129, 128, 64], [64, 64, 129, 127, 128, 65, 63], [300, 700]],
    200: [[1, 1, 60, 100], [200], [64, 64, 72]],
}


@pytest.mark.parametrize("p", [None, 0.1], ids=["nodrop", "drop0.1"])
@pytest.mark.parametrize("S", sorted(LAYOUTS))
def test_segments_vs_fp64(S, p):
    """Segment edges at 63 / 64 / 65 and 127 / 128 / 129 (the 64-row streamed and 128-row resident tiles), one-token
    segments and a trailing pad segment."""
    B, H = 3, 2
    qkv, dout = _case(B, S, H, seed=200 + S)
    seg = _seg_ids(LAYOUTS[S], S)
    out, lse, dqkv = _run(qkv, dout, H, seg_ids=seg, p=p)
    _check_fp64(qkv, dout, H, out, lse, dqkv, seg_ids=seg, p=p)


# ------------------------------------------------------------------------------------------------ exact answers
def _padded(qkv):
    """A copy of qkv with every head zero-padded to 128 columns: [B, S, 3, H, 128]."""
    pad = torch.zeros(*qkv.shape[:-1], 128, dtype=qkv.dtype, device=qkv.device)
    pad[..., :D] = qkv
    return pad


FORMS = {   # (key mask, segments, p)
    "causal": (False, False, None),
    "keymask": (True, False, None),
    "dropout": (False, False, 0.1),
    "keymask_dropout": (True, False, 0.1),
    "segments": (False, True, None),
}


@pytest.mark.parametrize("S", [129, 1024])
@pytest.mark.parametrize("form", sorted(FORMS))
def test_forward_is_the_d128_forward_on_zero_padded_heads(form, S):
    """O and LSE equal, bit for bit, those of the D = 128 kernel of the same form on zero-padded copies. Packed segments
    with p > 0 have no D = 128 kernel; their forward is covered by test_segments_vs_fp64."""
    masked, segmented, p = FORMS[form]
    B, H = 2, 3
    qkv, _ = _case(B, S, H, seed=300 + S)
    pad = _padded(qkv)
    mask = _key_mask(B, S) if masked else None
    scale = 1.0 / math.sqrt(D)
    outs = []
    for t in (qkv, pad):
        q, k, v = t[:, :, 0], t[:, :, 1], t[:, :, 2]
        if segmented:
            st, en = ops.segment_bounds(_seg_ids(LAYOUTS[1024][:B] if S == 1024 else [[64, 65], [1, 128]], S))
            outs.append(ops.sdpa_segments_fwd(q, k, v, scale, st, en, drop=_drop(p)))
        else:
            outs.append(ops.sdpa_fwd(q, k, v, scale, True, kv_mask=mask, drop=_drop(p)))
    torch.cuda.synchronize()
    (o96, l96), (o128, l128) = outs
    assert torch.equal(o96, o128[..., :D])
    assert torch.equal(l96, l128)


@pytest.mark.parametrize("form", sorted(FORMS) + ["segments_dropout"])
def test_backward_is_bit_identical_run_to_run(form):
    masked, segmented, p = FORMS.get(form, (False, True, 0.1))
    B, H, S = 2, 2, 1024
    qkv, dout = _case(B, S, H, seed=400)
    mask = _key_mask(B, S) if masked else None
    seg = _seg_ids(LAYOUTS[S][:B], S) if segmented else None
    a, b = _run(qkv, dout, H, mask, seg, p), _run(qkv, dout, H, mask, seg, p)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))


def test_one_token_segments_give_dropped_v_and_do():
    """Each query sees only itself: P = 1, so O = V Z / (1 - p) and dV = dO Z / (1 - p), Z the diagonal keep bit."""
    S, p, H = 200, 0.5, 2
    qkv, dout = _case(1, S, H, seed=5)
    out, lse, dqkv = _run(qkv, dout, H, seg_ids=torch.arange(S, device=DEV)[None], p=p)
    z = torch.from_numpy(R.attn_keep(SEED, BASE + SITE, 1, H, S, S, p)).diagonal(dim1=2, dim2=3)
    z = z.permute(0, 2, 1)[..., None].to(DEV)
    assert 0 < int(z.sum()) < z.numel()
    two = torch.tensor(2.0)   # 1 / (1 - 0.5): exact
    assert torch.equal(out, torch.where(z, qkv[:, :, 2].float() * two.to(DEV), 0.0).to(torch.bfloat16))
    assert torch.equal(dqkv[:, :, 2], torch.where(z, dout.float() * two.to(DEV), 0.0).to(torch.bfloat16))


# ------------------------------------------------------------------------------------------------ write footprint
@pytest.mark.parametrize("form", sorted(FORMS) + ["segments_dropout"])
def test_writes_stay_inside_each_head(form):
    """The attention runs on heads 1 and 2 of a 4-head packed tensor: O goes into a slice of a 4-head buffer and dq / dk /
    dv into the matching slices of one packed dqkv. The footprint guards check that every other byte (heads 0 and 3,
    and the columns past each head's 96, which a 128-wide store would reach) is untouched and that every declared byte
    is written."""
    masked, segmented, p = FORMS.get(form, (False, True, 0.1))
    B, S = 2, 200
    qkv, dout = _case(B, S, 2, seed=500, heads_total=4)
    q, k, v = (qkv[:, :, i, 1:3] for i in range(3))
    scale = 1.0 / math.sqrt(D)
    o_all = torch.zeros(B, S, 4, D, dtype=torch.bfloat16, device=DEV)
    dqkv = torch.randn(qkv.shape, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).to(DEV)
    dq, dk, dv = (dqkv[:, :, i, 1:3] for i in range(3))
    mask = _key_mask(B, S) if masked else None
    if segmented:
        st, en = ops.segment_bounds(_seg_ids([[64, 65, 71], [1, 199]], S))
        out, lse = F.check_footprint("sdpa_segments_fwd", ops.sdpa_segments_fwd, (q, k, v, scale, st, en),
                                     dict(out=o_all[:, :, 1:3], drop=_drop(p)))
        F.check_footprint("sdpa_segments_bwd", ops.sdpa_segments_bwd,
                          (q, k, v, out, dout, lse, scale, st, en, dq, dk, dv), dict(drop=_drop(p)))
    else:
        out, lse = F.check_footprint("sdpa_fwd", ops.sdpa_fwd, (q, k, v, scale, True),
                                     dict(kv_mask=mask, out=o_all[:, :, 1:3], drop=_drop(p)))
        F.check_footprint("sdpa_bwd", ops.sdpa_bwd, (q, k, v, out, dout, lse, scale, True, dq, dk, dv),
                          dict(kv_mask=mask, drop=_drop(p)))
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all()


# ------------------------------------------------------------------------------------------------ refusals
def test_head_dim_96_refuses_other_forms_and_runs_causal_segments_without_drop():
    B, S, H = 1, 128, 2
    qkv, _ = _case(B, S, H, seed=7)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    st, en = ops.segment_bounds(torch.zeros((B, S), dtype=torch.int64, device=DEV))
    rel = torch.zeros(H, 2 * S - 1, dtype=torch.float32, device=DEV)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_fwd(q, k, v, 0.1, False)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_fwd(q, k, v, 0.1, True, rel_bias=rel)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_fwd(q, k, v, 0.1, False, drop=_drop(0.1))
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, causal=False)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, rel_bias=rel)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_segments_fwd(q, k, v, 0.1, st, en, causal=False, kv_bounds=(st, en))
    lse = torch.zeros(B, H, S, dtype=torch.float32, device=DEV)
    d = torch.empty_like(q)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_bwd(q, k, v, q, q, lse, 0.1, False, d, d, d)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_bwd(q, k, v, q, q, lse, 0.1, True, d, d, d, rel_bias=rel)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_segments_bwd(q, k, v, q, q, lse, 0.1, st, en, d, d, d, causal=False)
    # causal segments without a drop run at head_dim 96: the kernels a Dropout(0.0) selects, bit for bit
    qkv, dout = _case(B, S, H, seed=8)
    seg = _seg_ids([[60, 68]], S)
    for x, y in zip(_run(qkv, dout, H, seg_ids=seg), _run(qkv, dout, H, seg_ids=seg, p=0.0)):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))
