"""Fused attention parity at the edges the models reach: causal attention with key padding (GPT-2 training, LLaMA's
left-padded prefill), KV-cache decode, sequences shorter than one tile, the relative-position bias gradient at batch >= 16,
and backward determinism.

Reference: softmax(scale q.k^T (+ bias), masked) v in fp32 on the same bf16 inputs, with autograd for the gradients. It is
built without NaN: a query row whose keys are all masked gets finite dummy scores and its probabilities are zeroed, and
only rows that see at least one key are compared numerically. The kernel's convention for a fully-masked row is pinned
exactly: O = 0, lse = +inf, dq = 0; a masked key gets dk = dv = 0.
Tolerance model, as in test_attention_gpu.py: P is rounded to bf16 before the PV product and O is stored in bf16, so O is
within 2e-2 of the reference on values of O(1) and lse within 2e-3; the gradients also round P and dS to bf16 before their
second GEMMs (3e-2 relative to the largest gradient).
Gradient buffers are views of NaN-filled packed buffers with guard rows and guard head slots (tests/guards.py).
"""
import math

import pytest
import torch

from guards import Guarded, bits

pytestmark = pytest.mark.gpu

from fsb200 import ops  # noqa: E402

DEV = "cuda"


def _randn(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _allowed(B, Sq, Sk, causal, kv_mask):
    ok = torch.ones(B, 1, Sq, Sk, dtype=torch.bool, device=DEV)
    if causal:
        ok &= torch.ones(Sq, Sk, dtype=torch.bool, device=DEV).tril()
    if kv_mask is not None:
        ok &= kv_mask.bool()[:, None, None, :]
    return ok


def _ref(q, k, v, scale, causal, kv_mask=None, rel=None):
    """q, k, v fp32 [B, S, H, D] (may require grad). Returns (O, natural-log lse, row_live [B, H, Sq])."""
    B, Sq, H, _ = q.shape
    Sk = k.shape[1]
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    if rel is not None:
        qi = torch.arange(Sq, device=DEV)[:, None]
        ki = torch.arange(Sk, device=DEV)[None, :]
        s = s + rel[:, ki - qi + Sq - 1][None]
    ok = _allowed(B, Sq, Sk, causal, kv_mask).expand(B, H, Sq, Sk)
    live = ok.any(-1)
    s = torch.where(ok, s, torch.full_like(s, float("-inf")))
    s = torch.where(live[..., None], s, torch.zeros_like(s))           # dummy finite scores for fully-masked rows
    p = torch.softmax(s, -1) * live[..., None]
    return torch.einsum("bhqk,bkhd->bqhd", p, v), torch.logsumexp(s, -1), live


def _packed(B, S, H, D):
    """NaN-filled [pad + B*S + pad, H, 3, D] buffer; slot 1 of each head is the [B, S, H, D] view, slots 0 and 2 and the
    pad rows are guards."""
    pad = 2
    buf = torch.full((B * S + 2 * pad, H, 3, D), float("nan"), dtype=torch.bfloat16, device=DEV)
    return Guarded(buf, lambda t: t[pad:pad + B * S].view(B, S, H, 3, D)[:, :, :, 1])


def _bwd_into_guards(q, k, v, out, dout, lse, scale, causal, kv_mask=None, rel=None, drel=None):
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    dq, dk, dv = _packed(B, Sq, H, D), _packed(B, Sk, H, D), _packed(B, Sk, H, D)
    ops.sdpa_bwd(q, k, v, out, dout, lse, scale, causal, dq.view, dk.view, dv.view, kv_mask=kv_mask, rel_bias=rel,
                 drel_bias=drel)
    return dq, dk, dv


def _check_grads(dq, dk, dv, qf, kf, vf, live, kv_mask, what):
    """Numerical comparison on the meaningful rows; exact zeros where nothing flows."""
    for name, g in (("dq", dq), ("dk", dk), ("dv", dv)):
        g.check(f"{what} {name}")
    live_q = live.permute(0, 2, 1)                                     # [B, Sq, H]
    assert torch.equal(dq.view[~live_q].float(), torch.zeros_like(dq.view[~live_q].float())), \
        f"{what}: dq of a fully-masked query row is not exactly 0"
    if kv_mask is not None:
        dead = ~kv_mask.bool()
        for name, g in (("dk", dk), ("dv", dv)):
            assert not g.view[dead].float().abs().gt(0).any(), f"{what}: {name} of a masked key is not exactly 0"
    for name, got, want, sel in (("dq", dq.view, qf.grad, live_q), ("dk", dk.view, kf.grad, None),
                                 ("dv", dv.view, vf.grad, None)):
        got = got.float()
        if sel is not None:
            got, want = got[sel], want[sel]
        err = (got - want).abs().max().item() if got.numel() else 0.0
        tol = 3e-2 * max(1.0, want.abs().max().item() if want.numel() else 0.0)
        assert err < tol, f"{what} {name}: max err {err} (tol {tol})"


def _check_fwd(out, lse, ref, ref_lse, live, what):
    live_q = live.permute(0, 2, 1)
    assert not torch.isnan(out.float()).any() and not torch.isnan(lse).any(), f"{what}: NaN in O or lse"
    assert torch.equal(out[~live_q].float(), torch.zeros_like(out[~live_q].float())), \
        f"{what}: O of a fully-masked row is not exactly 0"
    assert torch.isposinf(lse[~live]).all(), f"{what}: lse of a fully-masked row is not +inf"
    err = (out.float()[live_q] - ref[live_q]).abs().max().item()
    assert err < 2e-2, f"{what}: max |O - ref| = {err}"
    lerr = (lse[live] * math.log(2.0) - ref_lse[live]).abs().max().item()
    assert lerr < 2e-3, f"{what}: max |lse - ref| = {lerr}"


def _run_case(q, k, v, scale, causal, kv_mask, what, g):
    B, Sq, H, D = q.shape
    out, lse = ops.sdpa_fwd(q, k, v, scale, causal, kv_mask=kv_mask)
    qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
    ref, ref_lse, live = _ref(qf, kf, vf, scale, causal, kv_mask)
    _check_fwd(out, lse, ref.detach(), ref_lse.detach(), live, what)
    dout = _randn(B, Sq, H, D, g=g)
    ref.backward(dout.float())
    dq, dk, dv = _bwd_into_guards(q, k, v, out, dout, lse, scale, causal, kv_mask)
    _check_grads(dq, dk, dv, qf, kf, vf, live, kv_mask, what)
    again = _bwd_into_guards(q, k, v, out, dout, lse, scale, causal, kv_mask)
    for name, x, y in zip(("dq", "dk", "dv"), (dq, dk, dv), again):
        assert torch.equal(bits(x.buf), bits(y.buf)), f"{what}: {name} differs between two identical backward calls"


# ------------------------------------------------------------------------------------------------------------- B.1
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("S", [77, 200, 1024])
def test_causal_with_key_padding(S, D):
    """Batch row 0 unpadded, row 1 right-padded (GPT-2 training: causal + padding mask), row 2 left-padded (LLaMA prefill:
    its first query rows see no key at all)."""
    g = torch.Generator().manual_seed(S * 7 + D)
    B, H = 3, 2
    qkv = _randn(B, S, 3, H, D, g=g)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    mask = torch.ones(B, S, dtype=torch.uint8, device=DEV)
    mask[1, S - S // 3:] = 0
    mask[2, :S // 4 + 1] = 0
    _run_case(q, k, v, 1.0 / math.sqrt(D), True, mask, f"causal+padding S={S} D={D}", g)


# ------------------------------------------------------------------------------------------------------------- B.2
@pytest.mark.parametrize("Sq", [1, 3])
@pytest.mark.parametrize("Skv", [37, 129, 2048])
def test_kv_cache_decode(Sq, Skv):
    """LLaMA decode: q from the packed QKV projection ([B, Sq, H, 3, hn], slot 0), keys / values from a separate
    contiguous cache [B, Skv, H, hn]; not causal; the mask hides each row's left padding and the unwritten tail."""
    g = torch.Generator().manual_seed(Sq * 10000 + Skv)
    B, H, D = 3, 4, 128
    qkv = _randn(B, Sq, H, 3, D, g=g)
    q = qkv[:, :, :, 0]
    kc, vc = _randn(B, Skv, H, D, g=g), _randn(B, Skv, H, D, g=g)
    filled = max(1, Skv - Skv // 4)
    mask = torch.zeros(B, Skv, dtype=torch.uint8, device=DEV)
    for b, left in enumerate((0, 1, Skv // 3)):
        mask[b, min(left, filled - 1):filled] = 1
    _run_case(q, kc, vc, 1.0 / math.sqrt(D), False, mask, f"decode Sq={Sq} Skv={Skv}", g)


# ------------------------------------------------------------------------------------------------------------- B.3
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("S", [1, 8, 63, 64, 65, 129])
def test_short_sequences(S, causal, D):
    """Sequences shorter than (or just past) one 64-key / 128-query tile."""
    g = torch.Generator().manual_seed(S * 4 + D + int(causal))
    B, H = 2, 2
    qkv = _randn(B, S, H, 3, D, g=g)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    _run_case(q, k, v, 1.0 / math.sqrt(D), causal, None, f"S={S} causal={causal} D={D}", g)


# ------------------------------------------------------------------------------------------------------------- B.4
@pytest.mark.parametrize("causal,masked", [(True, False), (False, True)])
def test_rel_bias_gradient_large_batch(causal, masked):
    """B = 18 spreads over 16 batch splits in the bias-gradient reduction, two of which hold two batches; Sq = Sk = 200
    gives two query tiles. drel is accumulated onto prior content and is bit-identical on a second run. The reference
    drel is autograd of the fp32 formula; the kernel sums fp32 dS (before its bf16 rounding) along diagonals, so only P's
    ex2.approx and the bf16 inputs separate the two (2e-2 relative, as in test_attention_gpu.py)."""
    g = torch.Generator().manual_seed(18 + int(causal))
    B, S, H, D = 18, 200, 2, 64
    q, k = _randn(B, S, H, D, g=g, scale=0.5), _randn(B, S, H, D, g=g, scale=0.5)
    v = _randn(B, S, H, D, g=g)
    rel = (torch.randn(H, 2 * S - 1, generator=g) * 1.5).to(DEV)
    mask = None
    if masked:
        mask = torch.ones(B, S, dtype=torch.uint8, device=DEV)
        for b in range(B):
            mask[b, S - 7 * b - 1:] = 0
    out, lse = ops.sdpa_fwd(q, k, v, 1.0, causal, kv_mask=mask, rel_bias=rel)
    qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
    relf = rel.clone().requires_grad_(True)
    ref, ref_lse, live = _ref(qf, kf, vf, 1.0, causal, mask, relf)
    _check_fwd(out, lse, ref.detach(), ref_lse.detach(), live, "rel bias fwd")
    dout = _randn(B, S, H, D, g=g)
    ref.backward(dout.float())
    drel = torch.full_like(rel, 0.25)
    dq, dk, dv = _bwd_into_guards(q, k, v, out, dout, lse, 1.0, causal, mask, rel, drel)
    _check_grads(dq, dk, dv, qf, kf, vf, live, mask, "rel bias")
    want = relf.grad + 0.25
    err = (drel - want).abs().max().item()
    assert err < 2e-2 * max(1.0, want.abs().max().item()), f"drel: {err} vs max {want.abs().max().item()}"
    drel2 = torch.full_like(rel, 0.25)
    _bwd_into_guards(q, k, v, out, dout, lse, 1.0, causal, mask, rel, drel2)
    assert torch.equal(drel, drel2), "drel differs between two identical backward calls"


# ------------------------------------------------------------------------------------------------------------- B.5
def test_unsupported_head_dim_is_rejected():
    g = torch.Generator().manual_seed(0)
    q = _randn(1, 64, 2, 96, g=g)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_fwd(q, q, q, 0.1, False)
    lse = torch.zeros(1, 2, 64, dtype=torch.float32, device=DEV)
    d = torch.empty_like(q)
    with pytest.raises(RuntimeError, match="head_dim"):
        ops.sdpa_bwd(q, q, q, q, q, lse, 0.1, False, d, d, d)
