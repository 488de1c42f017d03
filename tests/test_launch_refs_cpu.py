"""The launch checkers of tests/launch_refs.py, proven on the CPU: for every op the reference agrees with torch autograd of
the fp64 forward (the bf16 rounding of the autograd result is accepted, at bounds about one ulp wide), and the bound
rejects the faults a kernel makes: one 64 x 64 block replaced by its neighbour's values, one row dropped from a column
sum, one 128-deep k-block missing from a GEMM, one head's O swapped with another's, one row's term dropped from a norm
backward. The census on the GPU (test_workload_launches_gpu.py) is only as strong as these proofs.
"""
import math

import pytest
import torch

import launch_refs as R

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
