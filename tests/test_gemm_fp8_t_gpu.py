"""GPU: fsb_gemm_fp8_t, the FP8 GEMM with a transposed store (`ops.gemm_fp8(..., store_transposed=True)`), which writes a
GPT-2 Conv1D's [in, out] weight gradient.

Bit for bit the transpose of fsb_gemm_fp8 on the same operands: at the C2 (hidden 768, 32 x 1024 tokens) and 3.5B (hidden
3072, 4 x 1024 tokens) weight-gradient shapes, with ragged m and n, with `accumulate` over a random old D, and into a
strided view. Exact on the integer operands of tests/fp8_ref.py, against fp64. A sentinel-filled buffer around D keeps its
sentinels. The refusals."""
import numpy as np
import pytest
import torch

from fp8_ref import encode, exact_operands
from fsb200 import lib as L
from fsb200 import ops

pytestmark = pytest.mark.gpu

E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
SENTINEL = -3.140625   # exact in bf16


def _codes(m, n, k, seed):
    """dy^T e5m2 codes [m, k] and x^T e4m3 codes [n, k] with their scales, as Fp8Conv1D's weight gradient reads them."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    # the quantiser takes multiples of 16: cast wider tensors and keep the first m / n rows of the codes
    dy = (torch.randn((k, m + (-m) % 16), device="cuda", generator=g) * 1e-3).to(torch.bfloat16)
    x = torch.randn((k, n + (-n) % 16), device="cuda", generator=g).to(torch.bfloat16)
    _, a, sa = ops.fp8_quantize(dy, "e5m2", rowwise=False, colwise=True)
    _, b, sb = ops.fp8_quantize(x, "e4m3", rowwise=False, colwise=True)
    return a[:m].contiguous(), sa, b[:n].contiguous(), sb


# (m, n, k) = (out, in, tokens): every C2 / 3.5B Conv1D's weight gradient, then ragged edges
@pytest.mark.parametrize("m,n,k", [
    (3 * 768, 768, 32768), (768, 768, 32768), (3072, 768, 32768), (768, 3072, 32768),          # C2: c_attn, c_proj, c_fc, mlp
    (3 * 3072, 3072, 4096), (3072, 3072, 4096), (12288, 3072, 4096), (3072, 12288, 4096),     # 3.5B
    (200, 136, 1040), (8, 1, 16), (136, 77, 256), (1000, 300, 512)])                           # ragged m / n
def test_equals_gemm_fp8_transposed(m, n, k):
    a, sa, b, sb = _codes(m, n, k, seed=m + 7 * n + k)
    d = ops.gemm_fp8(a, sa, b, sb, store_transposed=True)
    assert d.shape == (n, m)
    if n % 8 == 0:
        assert torch.equal(d, ops.gemm_fp8(a, sa, b, sb).t())
    else:   # fsb_gemm_fp8 needs n % 8 == 0: compare on n padded with zero rows of B
        bp = torch.zeros((n + (-n) % 8, k), dtype=E4, device="cuda")
        bp[:n] = b
        assert torch.equal(d, ops.gemm_fp8(a, sa, bp, sb)[:, :n].t())


@pytest.mark.parametrize("m,n,k", [(768, 3072, 4096), (200, 136, 1040), (136, 77, 256)])
def test_accumulate_into_a_strided_view_equals_gemm_fp8(m, n, k):
    """D (+)= into a view with ldd > m inside a sentinel-filled buffer: equal to gemm_fp8 accumulating onto D^T, and nothing
    outside the view changes."""
    a, sa, b, sb = _codes(m, n, k, seed=5 * m + n)
    g = torch.Generator(device="cuda").manual_seed(9)
    old = torch.randn((n, m), device="cuda", generator=g).to(torch.bfloat16) * 1e-2
    big = torch.full((n + 3, m + 40), SENTINEL, dtype=torch.bfloat16, device="cuda")
    d = big[1:1 + n, 16:16 + m]
    d.copy_(old)
    ops.gemm_fp8(a, sa, b, sb, out=d, accumulate=True, store_transposed=True)
    if n % 8 == 0:
        want = old.t().contiguous()
        ops.gemm_fp8(a, sa, b, sb, out=want, accumulate=True)
        assert torch.equal(d, want.t())
    outside = big.clone()
    outside[1:1 + n, 16:16 + m] = SENTINEL
    assert (outside == SENTINEL).all()
    ops.gemm_fp8(a, sa, b, sb, out=d, store_transposed=True)                      # overwrite: the product alone
    assert torch.equal(d, ops.gemm_fp8(a, sa, b, sb, store_transposed=True))
    assert (outside == SENTINEL).all()


def _exact(m, n, k, seed, ea=-3, eb=2):
    ai, bi = exact_operands(m, n, k, seed)
    a = torch.from_numpy(encode(ai.astype(np.float32), "e5m2")).cuda().view(E5)
    b = torch.from_numpy(encode(bi.astype(np.float32), "e4m3")).cuda().view(E4)
    sa, sb = torch.tensor([2.0 ** ea], device="cuda"), torch.tensor([2.0 ** eb], device="cuda")
    return a, sa, b, sb, (ai @ bi.T).astype(np.float64) * 2.0 ** (ea + eb)   # integers < 2^24 times a power of two


def _bf16(v):
    return torch.from_numpy(np.asarray(v, dtype=np.float32)).to(torch.bfloat16)


@pytest.mark.parametrize("m,n,k", [(16, 16, 16), (128, 128, 128), (200, 136, 1040), (8, 264, 4096), (296, 77, 2064)])
def test_exact_integer_codes(m, n, k):
    a, sa, b, sb, exact = _exact(m, n, k, seed=m + n + k)
    assert torch.equal(ops.gemm_fp8(a, sa, b, sb, store_transposed=True).cpu(), _bf16(exact.T))


def test_exact_accumulate_into_a_strided_view_with_sentinels():
    m, n, k = 136, 200, 640
    a, sa, b, sb, exact = _exact(m, n, k, seed=3)
    d0 = np.random.default_rng(4).integers(-64, 65, size=(n, m)) * 0.5   # the fp32 sum with the product stays exact
    big = torch.full((n + 2, m + 40), SENTINEL, dtype=torch.bfloat16, device="cuda")
    d = big[1:1 + n, 16:16 + m]
    d.copy_(_bf16(d0))
    ops.gemm_fp8(a, sa, b, sb, out=d, accumulate=True, store_transposed=True)
    assert torch.equal(d.cpu(), _bf16(exact.T + d0))
    big[1:1 + n, 16:16 + m] = SENTINEL
    assert (big == SENTINEL).all()


def test_fp64_reference_of_the_census():
    """The census's checker for the transposed store (tests/fp8_transposed_refs.py) accepts the kernel's result at a 3.5B
    c_fc shape, accumulating."""
    import fp8_transposed_refs as T
    import launch_refs as LR
    a, sa, b, sb = _codes(3072, 768, 1024, seed=2)
    out = torch.randn((768, 3072), device="cuda").to(torch.bfloat16)
    T.check_gemm_fp8_t(ops.gemm_fp8, LR.Bound("gemm_fp8 store_transposed"), a, sa, b, sb, out=out, accumulate=True)


def test_refusals():
    a, sa, b, sb = _codes(64, 32, 64, seed=1)
    a4 = ops.fp8_quantize(torch.ones((64, 64), dtype=torch.bfloat16, device="cuda"), "e4m3")[0]
    b5 = ops.fp8_quantize(torch.ones((32, 64), dtype=torch.bfloat16, device="cuda"), "e5m2")[0]
    for x, y in ((a4, b), (a, b5), (a4, b5)):
        with pytest.raises(RuntimeError, match=r"gemm_fp8_t: format pair .* only \(e5m2, e4m3\)"):
            ops.gemm_fp8(x, sa, y, sb, store_transposed=True)
    bias = torch.zeros(32, dtype=torch.bfloat16, device="cuda")
    aux = torch.zeros((64, 32), dtype=torch.bfloat16, device="cuda")
    for kw in (dict(bias=bias), dict(aux=aux), dict(epilogue=L.EPI_GELU_TANH)):
        with pytest.raises(RuntimeError, match="gemm_fp8_t: no bias, aux or epilogue"):
            ops.gemm_fp8(a, sa, b, sb, **kw, store_transposed=True)
    with pytest.raises(RuntimeError, match="m=12 must be a multiple of 8"):
        ops.gemm_fp8(a[:12].contiguous(), sa, b, sb, store_transposed=True)
    with pytest.raises(RuntimeError, match=r"out shape \(64, 32\) != \(32,64\)"):
        ops.gemm_fp8(a, sa, b, sb, out=torch.empty((64, 32), dtype=torch.bfloat16, device="cuda"), store_transposed=True)
    with pytest.raises(RuntimeError, match="accumulate needs an existing `out`"):
        ops.gemm_fp8(a, sa, b, sb, accumulate=True, store_transposed=True)
