"""The launch checkers of tests/launch_refs.py, proven on the CPU: for every op the reference agrees with torch autograd of
the fp64 forward (the bf16 rounding of the autograd result is accepted, at bounds about one ulp wide), and the bound
rejects the faults a kernel makes: one 64 x 64 block replaced by its neighbour's values, one row dropped from a column
sum, one 128-deep k-block missing from a GEMM, one head's O swapped with another's, one row's term dropped from a norm
backward. The dropout, quantisation, FP8 and decode checkers reject the mask of site + 1, a mask transposed in (q, k),
a mask without its 1 / (1 - p), a stream that lost its high word, an off-by-one counter, kv_append at slot kv_len,
attn_decode reading one slot past kv_len, kv_reorder writing past kv_len or gathering another layer, the neighbouring
channel's or group's scale, and an FP8 scale used uninverted. The censuses on the GPU (test_workload_launches_gpu.py,
test_path_launches_gpu.py) are only as strong as these proofs.
"""
import math

import numpy as np
import pytest
import torch

import fp8_ref
import int4_ref
import int8_ref
import launch_refs as R
import philox_ref

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _randn(*shape, seed=0, scale=1.0):
    return (torch.randn(*shape, generator=_g(seed)) * scale).to(BF16)


def _ok(fn, *args, **kw):
    b = R.Bound("cpu")
    fn(b, *args, **kw)
    assert b.worst <= 1.0
    return b.worst


def _rejects(fn, *args, **kw):
    with pytest.raises(AssertionError):
        fn(R.Bound("cpu"), *args, **kw)


def _swap_block(t, r0=64, c0=64):
    """Replace the 64 x 64 block at (r0, c0) by its left neighbour's values."""
    t = t.clone()
    t[r0:r0 + 64, c0:c0 + 64] = t[r0:r0 + 64, c0 - 64:c0].clone()
    return t


# ------------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("layout", [R.GEMM_NT, R.GEMM_NN, R.GEMM_TN])
@pytest.mark.parametrize("variant", ["plain", "bias", "gelu", "acc_f32", "acc_bf16"])
def test_gemm(layout, variant):
    M, N, K = 192, 256, 512
    A, B = _randn(M, K, seed=1), _randn(K, N, seed=2)
    a = A if layout != R.GEMM_TN else A.t().contiguous()
    b = B.t().contiguous() if layout == R.GEMM_NT else B
    bias = _randn(N, seed=3) if variant in ("bias", "gelu") else None
    epi = R.EPI_GELU_ERF if variant == "gelu" else R.EPI_NONE
    old = _randn(M, N, seed=4).to(F32 if variant == "acc_f32" else BF16) if variant.startswith("acc") else None
    odt = F32 if variant == "acc_f32" else BF16
    pre = A.double() @ B.double() + (bias.double() if bias is not None else 0.0)
    ref = R.act64(R.ACT_GELU_ERF, pre) if epi else pre
    ref = ref + (old.double() if old is not None else 0.0)
    aux = pre.to(BF16) if epi else None
    _ok(R.verify_gemm, layout, a, b, ref.to(odt), bias, epi, old, aux, aux.clone() if aux is not None else None)
    _ok(R.verify_gemm, layout, a, b, ref.to(odt), bias, epi, old, aux, None)
    _rejects(R.verify_gemm, layout, a, b, _swap_block(ref.to(odt)), bias, epi, old)
    lost = ref - A[:, 128:256].double() @ B[128:256].double()
    if epi:   # a lost k-block inside the activation
        lost = R.act64(R.ACT_GELU_ERF, pre - A[:, 128:256].double() @ B[128:256].double())
    _rejects(R.verify_gemm, layout, a, b, lost.to(odt), bias, epi, old)
    if aux is not None:
        bad = aux.clone()
        bad.view(torch.int16)[5, 7] += 1     # one bit of one element
        _rejects(R.verify_gemm, layout, a, b, ref.to(odt), bias, epi, old, bad, aux)


# ------------------------------------------------------------------------------------------------------------ norms
def _ln_stats(xs, eps, layer):
    xd = xs.double()
    if layer:
        mean = xd.mean(1)
        rstd = 1.0 / torch.sqrt((xd - mean[:, None]).pow(2).mean(1) + eps)
        return torch.stack([mean, rstd], 1).float()
    return (1.0 / torch.sqrt(xd.pow(2).mean(1) + eps)).float()


@pytest.mark.parametrize("layer", [False, True], ids=["rmsnorm", "layernorm"])
def test_norm_fwd(layer):
    rows, cols, eps = 130, 256, 1e-6
    x, r = _randn(rows, cols, seed=1), _randn(rows, cols, seed=2)
    w, beta = _randn(cols, seed=3, scale=0.3) + 1, _randn(cols, seed=4)
    xs = (x.float() + r.float()).to(BF16)
    st = _ln_stats(xs, eps, layer)
    xd = xs.double()
    if layer:
        y = torch.nn.functional.layer_norm(xd, (cols,), w.double(), beta.double(), eps).to(BF16)
    else:
        y = (xs.float() * st[:, None]).to(BF16) * w
    _ok(R.verify_norm_fwd, layer, x, r, w, beta if layer else None, eps, y, st, xs)
    _rejects(R.verify_norm_fwd, layer, x, r, w, beta if layer else None, eps, _swap_block(y), st, xs)
    bad = xs.clone(); bad[3, 5] = bad[3, 6] + 1
    _rejects(R.verify_norm_fwd, layer, x, r, w, beta if layer else None, eps, y, st, bad)


@pytest.mark.parametrize("layer", [False, True], ids=["rmsnorm", "layernorm"])
@pytest.mark.parametrize("wdt", [F32, BF16], ids=["f32", "bf16"])
def test_norm_bwd(layer, wdt):
    rows, cols, eps = 192, 256, 1e-6
    x, dy, dres = _randn(rows, cols, seed=1), _randn(rows, cols, seed=2), _randn(rows, cols, seed=5)
    w, beta = _randn(cols, seed=3, scale=0.3) + 1, _randn(cols, seed=4)
    st = _ln_stats(x, eps, layer)
    xd = x.double().requires_grad_(True)
    if layer:
        y = torch.nn.functional.layer_norm(xd, (cols,), w.double(), beta.double(), eps)
    else:
        y = xd * torch.rsqrt(xd.pow(2).mean(1, keepdim=True) + eps) * w.double()
    y.backward(dy.double())
    dx = (xd.grad + dres.double()).to(BF16)
    xw = (x.double() - st[:, 0:1].double()) * st[:, 1:2].double() if layer else (x.float() * st[:, None]).to(BF16).double()
    old = _randn(cols, seed=6).to(wdt)
    terms = dy.double() * xw
    dw = (terms.sum(0) + old.double()).to(wdt)
    db = (dy.double().sum(0) + old.double()).to(wdt) if layer else None
    args = (layer, dy, x, w, st, dres)
    _ok(R.verify_norm_bwd, *args, dx, dw, old, db, old if layer else None)
    _rejects(R.verify_norm_bwd, *args, _swap_block(dx), dw, old, db, old if layer else None)
    _rejects(R.verify_norm_bwd, *args, dx, (terms.sum(0) - terms[77] + old.double()).to(wdt), old, db,
             old if layer else None)
    if layer:
        _rejects(R.verify_norm_bwd, *args, dx, dw, old, (dy.double()[1:].sum(0) + old.double()).to(wdt), old)
    # one row's dropped term in the row sum mean(g xhat) of dx
    g = dy.double() * w.double()
    xh = (x.double() - (st[:, 0:1].double() if layer else 0.0)) * (st[:, 1:2] if layer else st[:, None]).double()
    core = g - xh * ((g * xh).sum(1, keepdim=True) - g[:, 40:41] * xh[:, 40:41]) / cols
    if layer:
        core = core - g.mean(1, keepdim=True)
    rstd = (st[:, 1:2] if layer else st[:, None]).double()
    bad = (rstd * core + dres.double()).to(BF16)
    _rejects(R.verify_norm_bwd, *args, bad, dw, old, db, old if layer else None)


# ------------------------------------------------------------------------------------------------------------- rope
@pytest.mark.parametrize("backward", [False, True])
def test_rope(backward):
    T, nh, hd = 96, 4, 128
    buf = _randn(T * nh * 3 * hd, seed=1)
    inv = 1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))
    fr = torch.arange(T).float()[:, None] * inv[None]
    cos, sin = fr.cos(), fr.sin()
    pos = torch.arange(T)
    args = (cos, sin, pos, nh, hd, 3 * nh * hd, 3 * hd, backward, hd)   # slot 1 (k) of the packed rows
    view = lambda t: R.rope_view(t, T, nh, hd, 3 * nh * hd, 3 * hd, hd)   # noqa: E731
    v = view(buf).double().requires_grad_(True)
    c = torch.cat([cos, cos], -1).double()[:, None]
    s = torch.cat([sin, sin], -1).double()[:, None]
    fwd = v * c + torch.cat([-v[..., hd // 2:], v[..., :hd // 2]], -1) * s
    if backward:   # the backward rotation is the transpose: J^T g through autograd
        g = view(buf).double()
        v2 = torch.zeros_like(g).requires_grad_(True)
        (v2 * c + torch.cat([-v2[..., hd // 2:], v2[..., :hd // 2]], -1) * s).backward(g)
        ref = v2.grad
    else:
        ref = fwd.detach()
    after = buf.clone()
    view(after).copy_(ref.to(BF16))
    _ok(R.verify_rope, buf, after, *args)
    bad = after.clone(); view(bad)[5, 2] = view(bad)[5, 3]
    _rejects(R.verify_rope, buf, bad, *args)
    bad = after.clone(); bad[0] += 1     # an element of slot 0 (q), outside the rotated heads
    _rejects(R.verify_rope, buf, bad, *args)


# ------------------------------------------------------------------------------------------------------ activations
@pytest.mark.parametrize("act", [R.ACT_SILU, R.ACT_GELU_TANH, R.ACT_GELU_ERF, R.ACT_TANH])
def test_activation_derivatives_match_autograd(act):
    x = torch.linspace(-8, 8, 4001, dtype=F64).requires_grad_(True)
    R.act64(act, x).sum().backward()
    assert torch.allclose(x.grad, R.dact64(act, x.detach()), rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("act", [R.ACT_SILU, R.ACT_GELU_TANH])
def test_glu(act):
    rows, cols = 128, 192
    gate, up, dout = _randn(rows, cols, seed=1), _randn(rows, cols, seed=2), _randn(rows, cols, seed=3)
    g, u = gate.double().requires_grad_(True), up.double().requires_grad_(True)
    out = R.act64(act, g) * u
    out.backward(dout.double())
    _ok(R.verify_glu_fwd, act, gate, up, out.detach().to(BF16))
    _rejects(R.verify_glu_fwd, act, gate, up, _swap_block(out.detach().to(BF16)))
    dg, du = g.grad.to(BF16), u.grad.to(BF16)
    _ok(R.verify_glu_bwd, act, dout, gate, up, dg, du)
    _rejects(R.verify_glu_bwd, act, dout, gate, up, _swap_block(dg), du)
    _rejects(R.verify_glu_bwd, act, dout, gate, up, dg, _swap_block(du))


@pytest.mark.parametrize("act", [R.ACT_GELU_TANH, R.ACT_GELU_ERF])
def test_act_and_bias_gradient(act):
    rows, cols = 192, 256
    x, dy = _randn(rows, cols, seed=1), _randn(rows, cols, seed=2)
    xd = x.double().requires_grad_(True)
    y = R.act64(act, xd)
    y.backward(dy.double())
    _ok(R.verify_act_fwd, act, x, y.detach().to(BF16))
    _rejects(R.verify_act_fwd, act, x, _swap_block(y.detach().to(BF16)))
    dx = xd.grad
    old = _randn(cols, seed=3).float()
    _ok(R.verify_act_bwd, act, dy, x, dx.to(BF16))
    dxs = dx.to(BF16).double()     # the bias gradient sums the stored bf16 dx
    _ok(R.verify_act_bwd, act, dy, x, dx.to(BF16), (dxs.sum(0) + old.double()).float(), old)
    _rejects(R.verify_act_bwd, act, dy, x, _swap_block(dx.to(BF16)))
    _rejects(R.verify_act_bwd, act, dy, x, dx.to(BF16), (dxs[1:].sum(0) + old.double()).float(), old)


@pytest.mark.parametrize("dt", [F32, BF16])
def test_colsum(dt):
    x = _randn(1000, 264, seed=1)
    old = _randn(264, seed=2).to(dt)
    _ok(R.verify_colsum, x, (x.double().sum(0) + old.double()).to(dt), old)
    _ok(R.verify_colsum, x, x.double().sum(0).to(dt))
    _rejects(R.verify_colsum, x, (x.double()[:999].sum(0)).to(dt))
    _rejects(R.verify_colsum, x, (x.double().sum(0) - x.double()[500]).to(dt))


# ------------------------------------------------------------------------------------------------------ elementwise
def test_elementwise():
    a, b = _randn(4096, seed=1), _randn(4096, seed=2)
    _ok(R.verify_add, a, b, (a.double() + b.double()).to(BF16))
    bad = (a.double() + b.double()).to(BF16); bad[100:164] = bad[36:100].clone()
    _rejects(R.verify_add, a, b, bad)
    acc = torch.randn(4096, generator=_g(3))
    _ok(R.verify_accumulate, acc, a, 0.5, False, (acc.double() + 0.5 * a.double()).float())
    _ok(R.verify_accumulate, None, a, 1.0, True, a.float())
    _rejects(R.verify_accumulate, acc, a, 0.5, False, (acc.double() + a.double()).float())
    _ok(R.verify_scale, a, 0.25, (a.double() * 0.25).to(BF16))
    _ok(R.verify_scale, a, 1.0, a.clone())
    _rejects(R.verify_scale, a, 0.25, (a.double() * 0.5).to(BF16))
    x32 = torch.randn(4096, generator=_g(4))
    _ok(R.verify_cast, x32, x32.to(BF16))
    bad = x32.to(BF16); bad.view(torch.int16)[9] += 1
    _rejects(R.verify_cast, x32, bad)


# -------------------------------------------------------------------------------------------------------- embedding
def test_embedding():
    V, cols, rows, S = 300, 256, 512, 128
    W, P, T = _randn(V, cols, seed=1), _randn(S, cols, seed=2), _randn(2, cols, seed=3)
    ids = torch.randint(0, V, (rows,), generator=_g(4))
    tt = torch.randint(0, 2, (rows,), generator=_g(5))
    _ok(R.verify_embedding_fwd, ids, W, None, None, None, None, 1, W[ids])
    bad = W[ids].clone(); bad[7] = W[(ids[7] + 1) % V]
    _rejects(R.verify_embedding_fwd, ids, W, None, None, None, None, 1, bad)
    Wd = W.double().requires_grad_(True)
    Pd = P.double().requires_grad_(True)
    t = torch.arange(rows)
    out = Wd[ids] + Pd[t % S] + T.double()[tt]
    _ok(R.verify_embedding_fwd, ids, W, None, P, tt, T, S, out.detach().to(BF16))
    _rejects(R.verify_embedding_fwd, ids, W, None, P, tt, T, S, _swap_block(out.detach().to(BF16)))
    dout = _randn(rows, cols, seed=6)
    out.backward(dout.double())
    old = _randn(V, cols, seed=7)
    new = (old.double() + Wd.grad).to(BF16)
    _ok(R.verify_embedding_bwd, ids, dout, old, new)
    _rejects(R.verify_embedding_bwd, ids, dout, old, _swap_block(new))
    lost = (old.double() + Wd.grad - torch.zeros_like(Wd.grad).index_add_(0, ids[3:4], dout.double()[3:4])).to(BF16)
    _rejects(R.verify_embedding_bwd, ids, dout, old, lost)       # one token's row dropped from its sum
    oldP = _randn(S, cols, seed=8)
    _ok(R.verify_embedding_bwd, None, dout, oldP, (oldP.double() + Pd.grad).to(BF16), S)
    _rejects(R.verify_embedding_bwd, None, dout, oldP, (oldP.double() + Pd.grad - dout.double()[S:2 * S]).to(BF16), S)


# --------------------------------------------------------------------------------------------------------- the loss
@pytest.mark.parametrize("dl_mode", ["out", "none"])
def test_softmax_xent(dl_mode):
    B, S, V = 4, 64, 1000
    logits = _randn(B * S, V, seed=1, scale=3.0)
    labels = torch.randint(0, V, (B * S,), generator=_g(2))
    labels[::5] = -100
    x = logits.double().view(B, S, V).requires_grad_(True)
    sl, lab = x[:, :-1].reshape(-1, V), labels.view(B, S)[:, 1:].reshape(-1)
    loss = torch.nn.functional.cross_entropy(sl, lab, ignore_index=-100)
    loss.backward()
    gs = 0.5
    n = torch.tensor(int((lab != -100).sum()), dtype=torch.int32)
    dl = (x.grad * gs).view(B * S, V).to(BF16) if dl_mode == "out" else None
    args = (logits, labels, S, 1, -100, gs)
    _ok(R.verify_softmax_xent, *args, loss.detach().float(), dl, n)
    _rejects(R.verify_softmax_xent, *args, loss.detach().float(), dl, n + 1)
    _rejects(R.verify_softmax_xent, *args, (loss.detach() * (1 + 1e-4)).float(), dl, n)
    if dl is not None:
        _rejects(R.verify_softmax_xent, *args, loss.detach().float(), _swap_block(dl), n)


# ---------------------------------------------------------------------------------------------------- the optimizer
@pytest.mark.parametrize("gdt,step,clip", [(BF16, 1, None), (F32, 7, 0.25)])
def test_adamw(gdt, step, clip):
    n = 128 * 128
    lr, b1, b2, eps, wd = 1e-3, 0.9, 0.95, 1e-8, 0.1
    p0 = torch.randn(n, generator=_g(1)) * 0.02
    m0 = torch.randn(n, generator=_g(2)) * 1e-3
    v0 = torch.rand(n, generator=_g(3)) * 1e-6
    grad = (torch.randn(n, generator=_g(4)) * 0.01).to(gdt)
    coef = None if clip is None else torch.tensor([clip])
    f = lambda v: float(torch.tensor(v, dtype=F32))   # noqa: E731  the fp32 scalars the C side receives
    prm = torch.nn.Parameter(p0.double())
    opt = torch.optim.AdamW([prm], lr=f(lr), betas=(f(b1), f(b2)), eps=f(eps), weight_decay=f(wd))
    st = opt.state[prm]
    prm.grad = grad.double() * (1.0 if clip is None else clip)
    opt.step()                       # torch initialises the state at the first step: set it, then redo
    st["exp_avg"].copy_(m0.double()); st["exp_avg_sq"].copy_(v0.double()); st["step"].fill_(step - 1)
    with torch.no_grad():
        prm.copy_(p0.double())
    opt.step()
    master, m, v = prm.detach().float(), st["exp_avg"].float(), st["exp_avg_sq"].float()
    args = (p0, m0, v0, grad)
    kw = dict(lr=lr, beta1=b1, beta2=b2, eps=eps, wd=wd, step=step, grad_scale=coef)
    _ok(R.verify_adamw, *args, master, m, v, master.to(BF16), **kw)
    _rejects(R.verify_adamw, *args, _swap_block(master.view(128, -1)).view(-1), m, v, None, **kw)
    _rejects(R.verify_adamw, *args, master, m, v, (master * 1.01).to(BF16), **kw)
    _rejects(R.verify_adamw, *args, master, _swap_block(m.view(128, -1)).view(-1), v, None, **kw)


def test_sumsq_and_clip():
    x = _randn(100000, seed=1)
    s = x.double().pow(2).sum()
    _ok(R.verify_sumsq, x, s.float().view(1))
    _ok(R.verify_sumsq, x, (s + 3.0).float().view(1), torch.tensor([3.0]))
    _rejects(R.verify_sumsq, x, (s - x.double()[7] ** 2 - x.double()[8] ** 2).float().view(1))
    _rejects(R.verify_sumsq, x, s.float().view(1), torch.tensor([3.0]))
    ss = torch.tensor([4.0])
    _ok(R.verify_clip_coef, ss, 1.0, torch.tensor([1.0 / (2.0 + 1e-6)]), torch.tensor([2.0]))
    _ok(R.verify_clip_coef, ss, 5.0, torch.tensor([1.0]), torch.tensor([2.0]))
    _rejects(R.verify_clip_coef, ss, 1.0, torch.tensor([0.5]), torch.tensor([2.0]))


# -------------------------------------------------------------------------------------------------------- attention
def _attn_case(causal, bias, mask, D=64):
    B, S, H = 2, 128, 3
    q = _randn(B, S, H, D, seed=1)
    k = _randn(B, S, H, D, seed=2)
    v = _randn(B, S, H, D, seed=3)
    rel = (torch.randn(H, 2 * S - 1, generator=_g(4)) * 2).float() if bias else None
    kvm = None
    if mask:
        kvm = torch.ones(B, S, dtype=torch.uint8)
        kvm[1, 100:] = 0
    return q, k, v, rel, kvm


def _attn_autograd(q, k, v, scale, causal, rel, kvm, dout):
    S = q.shape[1]
    qd, kd, vd = (R._bhsd(t).double().requires_grad_(True) for t in (q, k, v))
    s = scale * qd @ kd.transpose(-1, -2)
    relg = None
    if rel is not None:
        relg = rel.double().requires_grad_(True)
        i = torch.arange(S)
        s = s + relg[:, i[None, :] - i[:, None] + S - 1]
    if causal:
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
    if kvm is not None:
        s = s.masked_fill((kvm == 0)[:, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = torch.softmax(s, -1) @ vd
    o.backward(R._bhsd(dout).double())
    return o.detach(), lse.detach(), qd.grad, kd.grad, vd.grad, (relg.grad if relg is not None else None)


@pytest.mark.parametrize("causal,bias,mask", [(False, False, False), (True, False, False), (False, True, False),
                                              (False, False, True), (True, True, False)],
                         ids=["plain", "causal", "rel_bias", "kv_mask", "causal_rel_bias"])
def test_sdpa(causal, bias, mask):
    q, k, v, rel, kvm = _attn_case(causal, bias, mask)
    scale = 1.0 if bias else 1.0 / 8
    dout = _randn(*q.shape, seed=9)
    o, lse, dq, dk, dv, drel = _attn_autograd(q, k, v, scale, causal, rel, kvm, dout)
    O = R._bhsd(o).to(BF16)
    L2 = (lse / math.log(2.0)).float()
    fa = (q, k, v, scale, causal, kvm, rel)
    _ok(R.verify_sdpa_fwd, *fa, O, L2)
    Ow = O.clone(); Ow[:, :, 1] = O[:, :, 2]          # one head's O swapped with another's
    _rejects(R.verify_sdpa_fwd, *fa, Ow, L2)
    Ob = O.clone(); Ob[1, 64:128, 0] = O[1, 0:64, 0]  # one 64 x 64 block (64 queries x head_dim) replaced
    _rejects(R.verify_sdpa_fwd, *fa, Ob, L2)
    DQ, DK, DV = (R._bhsd(t).to(BF16) for t in (dq, dk, dv))
    old = torch.randn(rel.shape, generator=_g(5)).float() if bias else None
    new = (old.double() + drel).float() if bias else None
    ba = (q, k, v, O, dout, L2, scale, causal)
    _ok(R.verify_sdpa_bwd, *ba, DQ, DK, DV, kvm, rel, new, old)
    for i, t in enumerate((DQ, DK, DV)):
        bad = [DQ, DK, DV]
        tb = t.clone(); tb[0, 64:128, 1] = t[0, 0:64, 1]
        bad[i] = tb
        _rejects(R.verify_sdpa_bwd, *ba, *bad, kvm, rel, new, old)
    if bias:
        nb = new.clone(); nb[:, 100:164] = new[:, 36:100]
        _rejects(R.verify_sdpa_bwd, *ba, DQ, DK, DV, kvm, rel, nb, old)
        # one batch's (b = 1) contribution dropped from the bias gradient
        _, _, _, _, _, drel0 = _attn_autograd(q[:1], k[:1], v[:1], scale, causal, rel, None, dout[:1])
        _rejects(R.verify_sdpa_bwd, *ba, DQ, DK, DV, kvm, rel, (old.double() + drel0).float(), old)


def test_gemm_reference_in_small_chunks(monkeypatch):
    """The GEMM reference split into blocks of rows and columns (as a vocabulary-wide GEMM is on the GPU) accepts and
    rejects exactly what the one-block reference does."""
    M, N, K = 192, 256, 512
    A, B = _randn(M, K, seed=1), _randn(K, N, seed=2)
    bias = _randn(N, seed=3)
    pre = A.double() @ B.double() + bias.double()
    ref = R.act64(R.ACT_GELU_TANH, pre)
    aux = pre.to(BF16)
    monkeypatch.setattr(R, "CHUNK_BYTES", 8 * (2 * K + 14 * 64) * 48)   # 64 columns of B and 48 rows of A per block
    assert len(list(R._chunks(N, 8 * 2 * K))) > 1
    for layout in (R.GEMM_NT, R.GEMM_NN, R.GEMM_TN):
        a = A if layout != R.GEMM_TN else A.t().contiguous()
        b = B.t().contiguous() if layout == R.GEMM_NT else B
        _ok(R.verify_gemm, layout, a, b, ref.to(BF16), bias, R.EPI_GELU_TANH, None, aux, aux.clone())
        _rejects(R.verify_gemm, layout, a, b, _swap_block(ref.to(BF16), 128, 192), bias, R.EPI_GELU_TANH, None, aux, aux)
        lost = R.act64(R.ACT_GELU_TANH, pre - A[:, 128:256].double() @ B[128:256].double())
        _rejects(R.verify_gemm, layout, a, b, lost.to(BF16), bias, R.EPI_GELU_TANH, None, aux, aux)


# ---------------------------------------------------------------------------------------------------- dropout masks
SEED = 0x1234_5678_9ABC_DEF
HI = 2 ** 32 + 1        # a stream in the high word: base 2^32 - 5 plus site 6, as the GPU census draws them


def test_torch_philox_matches_numpy():
    """philox_ref's torch port gives the numpy masks bit for bit, in both layouts, for row / batch windows and for streams
    that carry into the high word."""
    for stream in (0, 5, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 3, 2 ** 45 + 2 ** 32 - 1):
        hk = philox_ref.hidden_keep(SEED, stream, 40, 88, 0.1)
        assert np.array_equal(philox_ref.hidden_keep_t(SEED, stream, range(0, 40), 88, 0.1).numpy(), hk)
        assert np.array_equal(philox_ref.hidden_keep_t(SEED, stream, range(7, 19), 88, 0.1).numpy(), hk[7:19])
        ak = philox_ref.attn_keep(SEED, stream, 3, 2, 40, 72, 0.1)
        assert np.array_equal(philox_ref.attn_keep_t(SEED, stream, range(0, 3), 2, 40, 72, 0.1).numpy(), ak)
        assert np.array_equal(philox_ref.attn_keep_t(SEED, stream, range(2, 3), 2, 40, 72, 0.1).numpy(), ak[2:])
    w = philox_ref.philox4x32_10_t((torch.tensor([0xFFFFFFFF, 0]), 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF, 0))
    wn = philox_ref.philox4x32_10((np.array([0xFFFFFFFF, 0]), 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF, 0))
    assert all(np.array_equal(a.numpy(), b.astype(np.int64)) for a, b in zip(w, wn))


def _spec(stream, p=0.1):
    return R.DropSpec(p, SEED, stream)


def _hmask(d, rows, cols, scaled=True):
    k = philox_ref.hidden_keep_t(d.seed, d.stream, range(rows), cols, d.p).double()
    return k * R.keep_scale(d.p) if scaled else k


FAULTS = {   # the masks a kernel could draw by mistake, as (spec, scaled) of the right spec d
    "site + 1": lambda d: (d._replace(stream=d.stream + 1), True),
    "no 1 / (1 - p)": lambda d: (d, False),
    "high word lost": lambda d: (d._replace(stream=d.stream & 0xFFFFFFFF), True),
}


def test_dropout_and_advance():
    rows, cols = 96, 264
    x = _randn(rows, cols, seed=1)
    d = _spec(HI + 1)
    ks = torch.tensor(R.keep_scale(d.p))
    good = torch.where(_hmask(d, rows, cols, False) > 0, x.float() * ks, torch.zeros(())).to(BF16)
    _ok(R.verify_dropout, x, d, good)
    for name, f in FAULTS.items():
        fd, scaled = f(d)
        _rejects(R.verify_dropout, x, d, (x.double() * _hmask(fd, rows, cols, scaled)).to(BF16))
    _ok(R.verify_dropout_advance, HI, 7, torch.tensor([HI]), torch.tensor([HI + 7]))
    _rejects(R.verify_dropout_advance, HI, 7, torch.tensor([HI]), torch.tensor([HI + 6]))
    _rejects(R.verify_dropout_advance, HI, 7, torch.tensor([HI + 1]), torch.tensor([HI + 7]))


@pytest.mark.parametrize("layer", [False, True], ids=["rmsnorm", "layernorm"])
def test_norm_dropout(layer):
    rows, cols, eps = 130, 256, 1e-6
    x, r, dy = _randn(rows, cols, seed=1), _randn(rows, cols, seed=2), _randn(rows, cols, seed=6)
    w, beta = _randn(cols, seed=3, scale=0.3) + 1, _randn(cols, seed=4)
    d = _spec(HI)
    ks = torch.tensor(R.keep_scale(d.p))

    def norm(xs):
        st = _ln_stats(xs, eps, layer)
        if layer:
            y = torch.nn.functional.layer_norm(xs.double(), (cols,), w.double(), beta.double(), eps).to(BF16)
        else:
            y = (xs.float() * st[:, None]).to(BF16) * w
        return y, st, xs
    xs = (torch.where(_hmask(d, rows, cols, False) > 0, x.float() * ks, torch.zeros(())) + r.float()).to(BF16)
    y, st, _ = norm(xs)
    args = (layer, x, r, w, beta if layer else None, eps)
    _ok(R.verify_norm_fwd, *args, y, st, xs, drop=d)
    for name, f in FAULTS.items():
        fd, scaled = f(d)
        _rejects(R.verify_norm_fwd, *args, *norm((x.double() * _hmask(fd, rows, cols, scaled) + r.double()).to(BF16)),
                 drop=d)
    # backward: dx of the sum (with dres), dbranch = M dx, through autograd of the fp64 norm
    xd = xs.double().requires_grad_(True)
    if layer:
        out = torch.nn.functional.layer_norm(xd, (cols,), w.double(), beta.double(), eps)
    else:
        out = xd * torch.rsqrt(xd.pow(2).mean(1, keepdim=True) + eps) * w.double()
    out.backward(dy.double())
    dx = xd.grad + r.double()               # r stands in for dres
    xw = (xs.double() - st[:, 0:1].double()) * st[:, 1:2].double() if layer else (xs.float() * st[:, None]).to(BF16).double()
    dw = (dy.double() * xw).sum(0).float()
    db = dy.double().sum(0).float() if layer else None
    bargs = (layer, dy, xs, w, st, r, dx.to(BF16), dw, None, db, None)
    _ok(R.verify_norm_bwd, *bargs, drop=d, dbranch=(dx * _hmask(d, rows, cols)).to(BF16))
    for name, f in FAULTS.items():
        fd, scaled = f(d)
        _rejects(R.verify_norm_bwd, *bargs, drop=d, dbranch=(dx * _hmask(fd, rows, cols, scaled)).to(BF16))


@pytest.mark.parametrize("act", [R.ACT_GELU_TANH, R.ACT_GELU_ERF])
def test_glu_dropout(act):
    rows, cols = 128, 192
    gate, up, dout = _randn(rows, cols, seed=1), _randn(rows, cols, seed=2), _randn(rows, cols, seed=3)
    d = _spec(HI + 2)

    def grads(m):
        g, u = gate.double().requires_grad_(True), up.double().requires_grad_(True)
        out = R.act64(act, g) * u * m
        out.backward(dout.double())
        return out.detach().to(BF16), g.grad.to(BF16), u.grad.to(BF16)
    out, dg, du = grads(_hmask(d, rows, cols))
    _ok(R.verify_glu_fwd, act, gate, up, out, d)
    _ok(R.verify_glu_bwd, act, dout, gate, up, dg, du, d)
    for name, f in FAULTS.items():
        fd, scaled = f(d)
        o_, dg_, du_ = grads(_hmask(fd, rows, cols, scaled))
        _rejects(R.verify_glu_fwd, act, gate, up, o_, d)
        _rejects(R.verify_glu_bwd, act, dout, gate, up, dg_, du_, d)


def _attn_dropout_autograd(q, k, v, scale, causal, rel, kvm, dout, m):
    S = q.shape[1]
    qd, kd, vd = (R._bhsd(t).double().requires_grad_(True) for t in (q, k, v))
    relg = rel.double().requires_grad_(True)
    i = torch.arange(S)
    s = scale * qd @ kd.transpose(-1, -2) + relg[:, i[None, :] - i[:, None] + S - 1]
    if causal:
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
    if kvm is not None:
        s = s.masked_fill((kvm == 0)[:, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = (torch.softmax(s, -1) * m) @ vd
    o.backward(R._bhsd(dout).double())
    grads = [qd.grad, kd.grad, vd.grad, relg.grad]
    return o.detach(), lse.detach(), grads


@pytest.mark.parametrize("causal", [False, True], ids=["rel_bias", "causal_rel_bias"])
def test_sdpa_dropout(causal):
    """Attention dropout with a rel_bias: with a padding mask (mT5's encoder) and with the causal flag (its decoder), where
    the bias at the offsets k - q > 0 is finite and masked by the flag (no NaN)."""
    B, S, H, D = 2, 64, 2, 64
    q, k, v = _randn(B, S, H, D, seed=1), _randn(B, S, H, D, seed=2), _randn(B, S, H, D, seed=3)
    rel = (torch.randn(H, 2 * S - 1, generator=_g(4)) * 2).float()
    kvm = None if causal else torch.ones(B, S, dtype=torch.uint8)
    if kvm is not None:
        kvm[1, 50:] = 0
    dout = _randn(B, S, H, D, seed=9)
    d = _spec(HI + 1)

    def mask(dd, scaled=True, transpose=False):
        z = philox_ref.attn_keep_t(dd.seed, dd.stream, range(B), H, S, S, dd.p).double()
        z = z.transpose(-1, -2) if transpose else z
        return z * R.keep_scale(dd.p) if scaled else z
    o, lse, (dq, dk, dv, drel) = _attn_dropout_autograd(q, k, v, 1.0, causal, rel, kvm, dout, mask(d))
    O, L2 = R._bhsd(o).to(BF16), (lse / math.log(2.0)).float()
    assert not torch.isnan(O.float()).any()
    fa = (q, k, v, 1.0, causal, kvm, rel)
    _ok(R.verify_sdpa_fwd, *fa, O, L2, d)
    old = torch.zeros_like(rel)
    ba = (q, k, v, O, dout, L2, 1.0, causal)
    DQ, DK, DV = (R._bhsd(t).to(BF16) for t in (dq, dk, dv))
    _ok(R.verify_sdpa_bwd, *ba, DQ, DK, DV, kvm, rel, drel.float(), old, d)
    faults = {"transposed (q, k)": mask(d, transpose=True)}
    faults.update({name: mask(*f(d)) for name, f in FAULTS.items()})
    for name, m in faults.items():
        o_, lse_, (dq_, dk_, dv_, drel_) = _attn_dropout_autograd(q, k, v, 1.0, causal, rel, kvm, dout, m)
        _rejects(R.verify_sdpa_fwd, *fa, R._bhsd(o_).to(BF16), L2, d)
        # the backward of a wrong mask, fed the right forward's O: dV alone already differs
        _rejects(R.verify_sdpa_bwd, *ba, DQ, DK, R._bhsd(dv_).to(BF16), kvm, rel, drel.float(), old, d)


def test_dropout_stream_invariants():
    """launch_census.dropout_stream_problems on synthetic logs: a consistent two-forward log passes; a too-small n, a
    counter that did not advance by n, an unused or doubly used site and a forward / backward mismatch are named."""
    from launch_census import dropout_stream_problems as problems
    n, b0 = 3, HI
    shape = (2, 4, 8, 8)

    def fb(base, site, kind=("sdpa_fwd", "sdpa_bwd"), p=0.1, sh=shape):
        return [(kind[0], base, site, p, SEED, sh), (kind[1], base, site, p, SEED, sh)]
    uses = []
    for base in (b0, b0 + n):
        uses += fb(base, 0) + fb(base, 1, ("dropout", "dropout"), sh=(16, 8)) + fb(base, 2, ("glu_fwd", "glu_bwd"))
    adv = [(b0, n), (b0 + n, n)]
    assert problems(adv, uses) == []
    assert any("not range(2)" in m for m in problems([(b0, 2), (b0 + 2, 2)], uses))            # n too small
    assert any("did not advance" in m for m in problems([(b0, n), (b0 + n - 1, n)], uses))       # off by one
    assert any("unused [2]" in m for m in problems(adv, [u for u in uses if u[2] != 2 or u[1] != b0]))
    assert any("drawn by" in m for m in problems(adv, uses + fb(b0, 0)[:1]))                    # a site drawn twice
    bad = [u if u[0] != "glu_bwd" or u[1] != b0 else (u[0], u[1], u[2], 0.2, *u[4:]) for u in uses]
    assert any("differ" in m for m in problems(adv, bad))                                        # p differs
    bad = [u if u[0] != "sdpa_bwd" or u[1] != b0 else ("layernorm_bwd_dropout", *u[1:]) for u in uses]
    assert any("drawn by" in m for m in problems(adv, bad))                                      # kinds differ


# ------------------------------------------------------------------------------------------------------------- FP8
@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_fp8_quantize_and_gemm(fmt):
    rows, cols = 64, 96
    x = _randn(rows, cols, seed=1, scale=0.01 if fmt == "e5m2" else 1.0)
    y, yt, sinv = fp8_ref.quantize(x.float().numpy(), fmt)
    dt = ops_fp8_dtype = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}[fmt]
    Y, YT = torch.from_numpy(y).view(dt), torch.from_numpy(yt).view(dt)
    S = torch.tensor([sinv], dtype=F32)
    _ok(R.verify_fp8_quantize, x, fmt, Y, YT, S)
    _ok(R.verify_fp8_quantize, x, fmt, None, YT, S)
    bad = Y.view(torch.uint8).clone(); bad[3, 5] ^= 1
    _rejects(R.verify_fp8_quantize, x, fmt, bad.view(dt), None, S)
    bad = YT.view(torch.uint8).clone(); bad[5, 3] ^= 1
    _rejects(R.verify_fp8_quantize, x, fmt, None, bad.view(dt), S)
    _rejects(R.verify_fp8_quantize, x, fmt, Y, YT, 1.0 / S)                 # the scale, not its inverse
    # the GEMM: out (+)= bf16((A B^T) sa sb) on the decoded codes
    w = _randn(80, cols, seed=2, scale=0.02)
    wq, _, ws = fp8_ref.quantize(w.float().numpy(), "e4m3")
    B8 = torch.from_numpy(wq).view(torch.float8_e4m3fn)
    SB = torch.tensor([ws], dtype=F32)
    a64, b64 = Y.float().double() * S.double(), B8.float().double() * SB.double()
    old = _randn(rows, 80, seed=3)
    for acc in (None, old):
        ref = a64 @ b64.t() + (acc.double() if acc is not None else 0.0)
        _ok(R.verify_gemm_fp8, Y, S, B8, SB, ref.to(BF16), acc)
        uninv = (Y.float().double() / S.double()) @ b64.t() + (acc.double() if acc is not None else 0.0)
        _rejects(R.verify_gemm_fp8, Y, S, B8, SB, uninv.to(BF16), acc)       # an FP8 scale used uninverted
        bad = ref.to(BF16); bad[:, 40:80] = bad[:, 0:40].clone()
        _rejects(R.verify_gemm_fp8, Y, S, B8, SB, bad, acc)
    _rejects(R.verify_gemm_fp8, Y, S, B8, SB, (a64 @ b64.t()).to(BF16), old)  # the accumulate term lost
    del ops_fp8_dtype


# --------------------------------------------------------------------------------------------- weight-only int8 / int4
def test_int8_quantize_and_gemm():
    n, k, m = 96, 256, 40
    w = _randn(n, k, seed=1, scale=0.05)
    w[7] = 0                                               # a zero row: s = 0, q = 0
    qn, sn = int8_ref.quantize(w.float().numpy())
    q, s = torch.from_numpy(qn), torch.from_numpy(sn)
    _ok(R.verify_quantize_w8, w, q, s)
    bad = q.clone(); bad[3, 9] += 1
    _rejects(R.verify_quantize_w8, w, bad, s)
    _rejects(R.verify_quantize_w8, w, q, s * (1 + 2 ** -20))
    a = _randn(m, k, seed=2)
    ref = (a.double() @ q.double().t()) * s.double()
    _ok(R.verify_gemm_w8a16, a, q, s, ref.to(BF16))
    nb = (a.double() @ q.double().t()) * s.double().roll(1)   # the neighbouring channel's scale
    _rejects(R.verify_gemm_w8a16, a, q, s, nb.to(BF16))


def test_int4_quantize_and_gemm():
    n, k, m = 64, 384, 24
    w = _randn(n, k, seed=1, scale=0.05)
    qn, sn = int4_ref.quantize(w.float().numpy())
    q, s = torch.from_numpy(int4_ref.pack(qn)), torch.from_numpy(sn).to(BF16)
    _ok(R.verify_quantize_w4, w, q, s)
    bad = q.clone(); bad[3, 9] ^= 0x10
    _rejects(R.verify_quantize_w4, w, bad, s)
    _rejects(R.verify_quantize_w4, w, q, s.roll(1, 1))
    W = torch.from_numpy(int4_ref.dequantize(qn, sn))
    assert torch.equal(R.unpack_w4(q, s).float(), W)
    a = _randn(m, k, seed=2)
    _ok(R.verify_gemm_w4a16, a, q, s, (a.double() @ W.double().t()).to(BF16))
    nb = torch.from_numpy(int4_ref.dequantize(qn, np.roll(sn, 1, axis=1)))   # the neighbouring group's scale
    _rejects(R.verify_gemm_w4a16, a, q, s, (a.double() @ nb.double().t()).to(BF16))


# --------------------------------------------------------------------------------------------------------- decoding
def _decode_case(B=3, H=2, D=64, cap=320):
    qd = _randn(B, H, D, seed=1)
    kc, vc = _randn(B, cap, H, D, seed=2), _randn(B, cap, H, D, seed=3)
    kvm = torch.ones(B, cap, dtype=torch.uint8)
    kvm[2, :40] = 0                                        # a left-padded row
    rel = torch.randn(H, 2 * cap - 1, generator=_g(4)).float()
    return qd, kc, vc, kvm, rel


def _decode_ref(q, kc, vc, L, scale, kvm, rel):
    cap = kc.shape[1]
    s = scale * torch.einsum("bhd,blhd->bhl", q.double(), kc[:, :L].double())
    if rel is not None:
        s = s + rel.double()[:, torch.arange(L) - (L - 1) + cap - 1][None]
    if kvm is not None:
        s = s.masked_fill((kvm[:, :L] == 0)[:, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1)
    return torch.einsum("bhl,blhd->bhd", torch.softmax(s, -1), vc[:, :L].double()), lse / math.log(2.0)


@pytest.mark.parametrize("variant", ["kv_mask", "rel_bias"])
def test_attn_decode(variant):
    q, kc, vc, kvm, rel = _decode_case()
    kvm = kvm if variant == "kv_mask" else None
    rel = rel if variant == "rel_bias" else None
    scale = 0.125
    L = 257
    o, lse = _decode_ref(q, kc, vc, L, scale, kvm, rel)
    _ok(R.verify_attn_decode, q, kc, vc, L, scale, kvm, rel, o.to(BF16), lse.float())
    o1, lse1 = _decode_ref(q, kc, vc, L + 1, scale, kvm, rel) if rel is None else (None, None)
    if rel is not None:   # one slot past kv_len, with the bias row of kv_len - 1
        cap = kc.shape[1]
        s = scale * q.double()[:, :, None, :].mul(kc[:, :L + 1].double().permute(0, 2, 1, 3)).sum(-1)
        s = s + rel.double()[:, torch.arange(L + 1) - (L - 1) + cap - 1][None]
        o1 = torch.einsum("bhl,blhd->bhd", torch.softmax(s, -1), vc[:, :L + 1].double())
        lse1 = torch.logsumexp(s, -1) / math.log(2.0)
    _rejects(R.verify_attn_decode, q, kc, vc, L, scale, kvm, rel, o1.to(BF16), lse.float())
    _rejects(R.verify_attn_decode, q, kc, vc, L, scale, kvm, rel, o.to(BF16), lse1.float())


def test_kv_append():
    B, cap, H, D = 3, 40, 2, 64
    kn, vn = _randn(B, H, D, seed=1), _randn(B, H, D, seed=2)
    kb, vb = _randn(B, cap, H, D, seed=3), _randn(B, cap, H, D, seed=4)
    mb = torch.zeros(B, cap, dtype=torch.uint8); mb[:, :20] = 1
    L = 21

    def appended(slot):
        k, v, m = kb.clone(), vb.clone(), mb.clone()
        k[:, slot], v[:, slot], m[:, slot] = kn, vn, 1
        return k, v, m
    _ok(R.verify_kv_append, kn, vn, L, kb, vb, mb, *appended(L - 1))
    _rejects(R.verify_kv_append, kn, vn, L, kb, vb, mb, *appended(L))         # slot kv_len instead of kv_len - 1
    k, v, m = appended(L - 1); m[0, 30] = 1
    _rejects(R.verify_kv_append, kn, vn, L, kb, vb, mb, k, v, m)               # a stray mask bit
    k, v, m = appended(L - 1); v[1, 3, 1, 7] += 1
    _rejects(R.verify_kv_append, kn, vn, L, kb, vb, mb, k, v, m)               # another V element changed
    _ok(R.verify_kv_append, kn, vn, cap + 1, kb, vb, mb, kb.clone(), vb.clone(), mb.clone())   # outside: no change


def test_kv_reorder():
    layers, rows, cap, slot = 3, 4, 24, 2 * 2 * 64
    src = _randn(layers, rows, cap, slot, seed=1)
    before = _randn(layers, rows, cap, slot, seed=2)
    index = torch.tensor([2, 2, 0, 3])
    L = 17
    want = before.clone(); want[:, :, :L] = src[:, index, :L]
    _ok(R.verify_kv_reorder, src, index, L, before, want)
    past = want.clone(); past[:, :, L] = src[:, index, L]
    _rejects(R.verify_kv_reorder, src, index, L, before, past)                # written past kv_len
    other = want.clone(); other[1, :, :L] = src[2][index, :L]
    _rejects(R.verify_kv_reorder, src, index, L, before, other)              # another layer's rows
