"""Parity of the training step's smaller kernels under the options the models pass: LayerNorm with a fused residual add
and its gradient, cross-entropy without the causal shift and with a loss scale, embeddings with positions and token types,
column sums over strided rows, AdamW with fp32 gradients and device scalars, and the fp32 / bf16 vector helpers.

Each test compares with the torch formula of what the model computes, in fp32 (fp64 for reductions) on the same bf16
inputs. Tolerance model, as in test_kernels_gpu.py: one bf16 rounding of an fp32 result (rtol ~2^-8) plus fp32
accumulation-order noise growing with sqrt(reduction length). Outputs that are passed in are views of NaN-filled (or, when
accumulated into, finite) buffers with guards (tests/guards.py).
"""
import math

import pytest
import torch

from guards import bits, guarded_1d, guarded_2d

pytestmark = pytest.mark.gpu

from fsb200 import lib as L, ops  # noqa: E402

DEV = "cuda"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _close(got, ref, atol, rtol, what=""):
    err = (got.double() - ref.double()).abs()
    bad = err > atol + rtol * ref.double().abs()
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} elements off; max err {err.max().item():.4g}"


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("rows,cols", [(1, 16384), (77, 768), (300, 1024)])
@pytest.mark.parametrize("wdt", [torch.float32, torch.bfloat16])
def test_layernorm_residual_and_dres(rows, cols, wdt):
    """GPT-2 / BERT main path: y = LN(x + residual) with the bf16 sum written out, and dx = LN'(dy) + dres, with dgamma /
    dbeta accumulated onto what the buffers already hold, in fp32 or bf16."""
    x, r = _rand(rows, cols, seed=1), _rand(rows, cols, seed=2)
    gamma = (1 + 0.1 * torch.randn(cols)).to(torch.bfloat16).to(DEV)
    beta = (0.1 * torch.randn(cols)).to(torch.bfloat16).to(DEV)
    eps = 1e-5
    n = rows * cols
    y, xs, st = guarded_1d(n, torch.bfloat16), guarded_1d(n, torch.bfloat16), guarded_1d(2 * rows, torch.float32)
    L.call("fsb_layernorm_fwd", x.data_ptr(), r.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.view.data_ptr(),
           xs.view.data_ptr(), st.view.data_ptr(), rows, cols, eps, _stream())
    for name, t in (("y", y), ("sum_out", xs), ("stats", st)):
        t.check(f"layernorm {name}")
    xs_ref = (x.float() + r.float()).to(torch.bfloat16)
    assert torch.equal(xs.view.view(rows, cols), xs_ref), "sum_out is not the bf16 sum x + residual"
    xf = xs_ref.double().requires_grad_(True)
    gf, bf = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    yref = torch.nn.functional.layer_norm(xf, (cols,), gf, bf, eps)
    _close(y.view.view(rows, cols), yref.detach(), 2e-2, 1e-2, "layernorm fwd")
    dy, dres = _rand(rows, cols, seed=3), _rand(rows, cols, seed=4)
    yref.backward(dy.double())
    g0 = guarded_1d(cols, wdt, fill=0.0, init=torch.full((cols,), 0.5))
    b0 = guarded_1d(cols, wdt, fill=0.0, init=torch.full((cols,), -0.25))
    dx = ops.layernorm_bwd(dy, xs.view.view(rows, cols), gamma, st.view.view(rows, 2), g0.view, b0.view, accumulate=True,
                           dres=dres)
    g0.check("dgamma", written=False)
    b0.check("dbeta", written=False)
    _close(dx, xf.grad + dres.double(), 3e-2, 2e-2, "layernorm dx + dres")
    wtol = 0.05 * math.sqrt(rows / 64)
    rt = 2e-2 if wdt == torch.float32 else 3e-2
    _close(g0.view, gf.grad + 0.5, wtol, rt, "dgamma accumulated")
    _close(b0.view, bf.grad - 0.25, wtol, rt, "dbeta accumulated")


# ----------------------------------------------------------------------------------------------------------- cross-entropy
def _xent_ref(logits, labels, S, shift, ignore=-100):
    V = logits.shape[1]
    lf = logits.double().view(-1, S, V).requires_grad_(True)
    lab = labels.view(-1, S)
    if shift:
        x, t = lf[:, :-shift].reshape(-1, V), lab[:, shift:].reshape(-1)
    else:
        x, t = lf.reshape(-1, V), lab.reshape(-1)
    n = int((t != ignore).sum())
    if n == 0:
        return torch.zeros((), dtype=torch.float64, device=DEV), torch.zeros_like(lf).view(-1, V), 0
    loss = torch.nn.functional.cross_entropy(x, t, ignore_index=ignore)
    loss.backward()
    return loss.detach(), lf.grad.view(-1, V), n


@pytest.mark.parametrize("V", [8, 21128, 250112])
@pytest.mark.parametrize("shift", [0, 1])
def test_softmax_xent_options(V, shift):
    """shift = 0 (BERT / T5 MLM) and 1 (causal LM); loss scale != 1; dlogits in place, into a separate buffer, or not at all;
    a row stride ld > V with guards in the padding columns; logits of magnitude ~80."""
    B, S = 2, 12
    rows = B * S
    g = torch.Generator().manual_seed(V + shift)
    logits = (torch.randn(rows, V, generator=g) * 20).clamp(-80, 80)
    logits[:, 3] = 80.0
    logits = logits.to(torch.bfloat16).to(DEV)
    labels = torch.randint(0, V, (rows,), generator=g).to(DEV)
    labels[5] = -100
    labels[0] = 3
    ref_loss, ref_grad, n = _xent_ref(logits, labels, S, shift)
    scale = 0.375
    # padded row stride, dlogits in place
    buf = guarded_2d(rows, V, torch.bfloat16, fill=float("nan"), init=logits, pad_rows=0, pad_cols=8)
    loss, dl, nv = ops.softmax_xent(buf.view, labels, S, shift=shift, grad_scale=scale)
    buf.check(f"xent in place V={V}")
    assert nv.item() == n
    assert abs(loss.item() - ref_loss.item()) < 2e-4 * max(1.0, abs(ref_loss.item())), (loss.item(), ref_loss.item())
    _close(buf.view, ref_grad * scale, 2e-5, 1.6e-2, "dlogits in place")
    # separate dlogits buffer: logits untouched
    sep = guarded_2d(rows, V, torch.bfloat16, pad_rows=2, pad_cols=0)   # same ld as the contiguous logits
    src = logits.clone()
    L.call("fsb_softmax_xent_fwd_bwd", src.data_ptr(), labels.data_ptr(), sep.view.data_ptr(),
           torch.empty(rows, device=DEV).data_ptr(), loss.data_ptr(), nv.data_ptr(), rows, V, V, S, shift, -100, scale,
           _stream())
    sep.check("separate dlogits")
    assert torch.equal(src, logits), "logits changed although dlogits is a separate buffer"
    assert torch.equal(bits(sep.view), bits(buf.view)), "separate dlogits differ from the in-place result"
    # no gradient at all: loss only
    src2 = logits.clone()
    loss2, dl2, _ = ops.softmax_xent(src2, labels, S, shift=shift, dlogits=None)
    assert dl2 is None and torch.equal(src2, logits)
    assert loss2.item() == loss.item()


def test_softmax_xent_all_ignored():
    """A batch whose labels are all ignore_index: loss 0, gradient exactly 0, nothing NaN."""
    rows, V = 16, 64
    logits = _rand(rows, V, seed=5)
    labels = torch.full((rows,), -100, dtype=torch.int64, device=DEV)
    for shift in (0, 1):
        work = logits.clone()
        loss, dl, nv = ops.softmax_xent(work, labels, 8, shift=shift, grad_scale=2.0)
        assert nv.item() == 0 and loss.item() == 0.0
        assert torch.equal(dl.float(), torch.zeros(rows, V, device=DEV))


# ----------------------------------------------------------------------------------------------------------- embeddings
def test_embedding_positions_and_token_types():
    """BERT: out[t] = W[ids[t]] + P[pos[t]] + T[token_type[t]] (explicit positions), and the learned-position backward
    dW[t % idx_mod] += dout[t] (ids = None)."""
    V, H, B, S, NT = 1000, 256, 3, 40, 2
    W, P, T = _rand(V, H, seed=1), _rand(512, H, seed=2), _rand(NT, H, seed=3)
    ids = torch.randint(0, V, (B * S,), device=DEV)
    pos = (torch.arange(S, device=DEV) + 5).repeat(B)
    tt = torch.randint(0, NT, (B * S,), device=DEV)
    out = ops.embedding_fwd(ids, W, pos=pos, P=P, token_type=tt, T=T, seq_len=S)
    ref = W[ids].double() + P[pos].double() + T[tt].double()
    _close(out, ref, 1e-2, 8e-3, "word + position + token type")
    dout = _rand(B * S, H, seed=4, scale=0.1)
    base = _rand(S, H, seed=5)
    dP = base.clone()
    ops.embedding_bwd(None, dout, dP, idx_mod=S)
    want = base.double() + dout.double().view(B, S, H).sum(0)
    # bf16 atomics: B additions, each rounded to bf16
    _close(dP, want, 1e-2, 2e-2, "position gradient, ids=None / idx_mod")


# ----------------------------------------------------------------------------------------------------------- colsum
@pytest.mark.parametrize("odt", [torch.float32, torch.bfloat16])
def test_colsum_strided_rows(odt):
    """Bias gradient over a row-strided view (ld > cols), written and accumulated, fp32 and bf16 out."""
    rows, cols = 777, 1032
    big = _rand(rows, cols + 64, seed=6)
    x = big[:, 16:16 + cols]
    ref = x.double().sum(0)
    out = guarded_1d(cols, odt)
    ops.colsum(x, out.view)
    out.check("colsum")
    tol = 1e-3 * math.sqrt(rows) if odt == torch.float32 else 0.3
    _close(out.view, ref, tol, 1e-2 if odt == torch.bfloat16 else 1e-5, "colsum")
    acc = guarded_1d(cols, odt, fill=0.0, init=torch.full((cols,), 3.0))
    ops.colsum(x, acc.view, accumulate=True)
    acc.check("colsum accumulate", written=False)
    _close(acc.view, ref + 3.0, tol, 1e-2 if odt == torch.bfloat16 else 1e-5, "colsum accumulate")


# ----------------------------------------------------------------------------------------------------------- AdamW
@pytest.mark.parametrize("mode", ["f32_grad", "grad_scale", "hyper"])
def test_adamw_options_match_torch_optim(mode):
    """fp32 gradients (ZeRO-2 accumulators), a device gradient scale (clip coefficient), and device hyper-parameters
    {lr, 1 - beta1^t, sqrt(1 - beta2^t)} in place of lr / step (CUDA-graph form), over several steps."""
    n = 4096 * 3 + 4
    gen = torch.Generator().manual_seed(7)
    p0 = torch.randn(n, generator=gen).to(DEV)
    master, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    p16 = guarded_1d(n, torch.bfloat16)
    ref = torch.nn.Parameter(p0.clone().double())
    lr, b1, b2, eps, wd = 3e-3, 0.9, 0.95, 1e-8, 0.1
    opt = torch.optim.AdamW([ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    for step in range(1, 6):
        g = torch.randn(n, generator=gen).to(DEV)
        coef = 0.5 + 0.1 * step
        if mode == "f32_grad":
            ref.grad = g.double()
            ops.adamw_flat(master, m, v, g, p16.view, lr, b1, b2, eps, wd, step)
        elif mode == "grad_scale":
            g16 = g.to(torch.bfloat16)
            ref.grad = g16.double() * torch.tensor(coef, dtype=torch.float32).double()
            ops.adamw_flat(master, m, v, g16, p16.view, lr, b1, b2, eps, wd, step,
                           grad_scale=torch.tensor(coef, dtype=torch.float32, device=DEV))
        else:
            ref.grad = g.double()
            hyper = torch.tensor([lr, 1 - b1 ** step, math.sqrt(1 - b2 ** step)], dtype=torch.float32, device=DEV)
            ops.adamw_flat(master, m, v, g, p16.view, 1e9, b1, b2, eps, wd, 0, hyper=hyper)
        opt.step()
        _close(master, ref.data, 1e-6, 1e-5, f"adamw {mode} step {step}")
    p16.check("param16")
    assert torch.equal(p16.view, master.to(torch.bfloat16))


# ----------------------------------------------------------------------------------------------------------- vector helpers
def test_sumsq_fp32_accumulate():
    x = torch.randn(8192 * 4 + 4, generator=torch.Generator().manual_seed(8)).to(DEV)
    out = torch.full((), 2.5, dtype=torch.float32, device=DEV)
    ops.sumsq(x, out, accumulate=True)
    ref = x.double().pow(2).sum().item() + 2.5
    assert abs(out.item() - ref) < 1e-5 * ref, (out.item(), ref)


def test_add_accumulate_scale_cast():
    n = 8 * 1237
    a, b = _rand(n, seed=9), _rand(n, seed=10)
    out = guarded_1d(n, torch.bfloat16)
    ops.add(a, b, out=out.view)
    out.check("add")
    assert torch.equal(out.view, (a.float() + b.float()).to(torch.bfloat16)), "add is not one rounding of the fp32 sum"
    init = torch.randn(n, generator=torch.Generator().manual_seed(11)).to(DEV)
    for overwrite in (False, True):
        acc = guarded_1d(n, torch.float32, fill=0.0, init=init)
        ops.accumulate(acc.view, a, scale=0.75, overwrite=overwrite)
        acc.check(f"accumulate overwrite={overwrite}", written=False)
        want = 0.75 * a.double() + (0 if overwrite else init.double())
        _close(acc.view, want, 1e-6, 1e-6, f"accumulate overwrite={overwrite}")
    for s in (1.0, -0.3125):
        x = guarded_1d(n, torch.bfloat16, fill=0.0, init=a)
        ops.scale_inplace(x.view, torch.tensor(s, device=DEV))
        x.check(f"scale {s}", written=False)
        assert torch.equal(x.view, (a.float() * s).to(torch.bfloat16)), f"scale_inplace by {s}"
    x32 = torch.randn(n, generator=torch.Generator().manual_seed(12)).to(DEV) * 100
    cast = guarded_1d(n, torch.bfloat16)
    ops.cast_f32_to_bf16(x32, out=cast.view)
    cast.check("cast")
    assert torch.equal(cast.view, x32.to(torch.bfloat16)), "cast is not round-to-nearest-even"
