"""GPU: the reference's own two CUDA ops (scaled_masked_softmax_cuda, scaled_upper_triang_masked_softmax_cuda) served by
libfsb200.so through the same Python module names and signatures. The reference's only stated tolerance for these kernels
is mean |diff| <= 1e-3 vs torch softmax (fused_kernels/tests/test_fused_kernels.py:97-104,197-204); we assert that AND an
elementwise bound of one bf16 ulp of the fp64 value (the kernel rounds its fp32 result once) plus a small absolute floor:
1e-6 * max|ref| in the forward (fp32 exp / sum); in the backward 1e-5 * the row's max |y| * (|dy| + |sum(dy * y)|), the
size of the two fp32 terms whose difference the kernel takes."""
import os
import sys

import pytest
import torch

from guards import assert_ulp_close, bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))

import scaled_masked_softmax_cuda as sms  # noqa: E402
import scaled_upper_triang_masked_softmax_cuda as suts  # noqa: E402


def _randn(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to("cuda")


def _check_bwd(dx, dy, y, scale, what):
    """dx against the fp64 formula on the kernel's own bf16 y (the reference kernel differentiates through it too)."""
    yy, g = y.double(), dy.double()
    dot = (g * yy).sum(-1, keepdim=True)
    want = scale * (g * yy - yy * dot)
    floor = 1e-5 * scale * (yy * (g.abs() + dot.abs())).amax(-1, keepdim=True)
    assert_ulp_close(dx, want, what, floor=floor)


@pytest.mark.parametrize("b,np_,sq,sk,mb", [(2, 4, 64, 64, 2), (1, 3, 128, 256, 1), (2, 2, 40, 2048, 1), (1, 2, 16, 1000, 1),
                                            (2, 3, 16, 8, 2), (2, 3, 16, 8, 1), (2, 3, 16, 264, 2), (2, 3, 12, 520, 1),
                                            (2, 3, 8, 1032, 2), (2, 3, 8, 2056, 1), (2, 3, 8, 4096, 2), (2, 3, 4, 4096, 1)])
def test_scaled_masked_softmax_fwd_bwd(b, np_, sq, sk, mb):
    """sk over every vectors-per-lane bucket up to the 4096 maximum, one mask per batch or one broadcast mask. Query rows
    0 and sq - 1 of the first mask are fully masked: the reference fills masked scores with -10000, not -inf, so those
    rows are exactly uniform (1 / sk) and their gradient is finite."""
    x = _randn(b, np_, sq, sk, scale=3, seed=sk + sq)
    g = torch.Generator().manual_seed(sk)
    mask = (torch.rand(mb, 1, sq, sk, generator=g) < 0.2)
    mask[0, 0, 0] = True
    mask[0, 0, sq - 1] = True
    mask = mask.to("cuda")
    scale = 0.125
    y = sms.forward(x, mask, scale)
    xf = x.float().requires_grad_(True)
    ref = torch.softmax((xf * scale).masked_fill(mask, -10000.0), dim=-1)     # fused_softmax.py mask_func semantics
    assert (y.float() - ref).abs().mean().item() <= 1e-3
    ref64 = torch.softmax(torch.where(mask, torch.tensor(-10000.0, dtype=torch.float64, device="cuda"), x.double() * scale),
                          dim=-1)
    assert_ulp_close(y, ref64, f"masked softmax fwd sk={sk}", floor=1e-6 * ref64.abs().max().item())
    full = mask.all(-1).expand(b, np_, sq)                                    # [b, np, sq] rows with every key masked
    assert full.sum().item() == (2 if mb == b else 2 * b) * np_
    uniform = torch.tensor(1.0 / sk, dtype=torch.float32).to(torch.bfloat16).to("cuda")
    assert torch.equal(bits(y[full]), bits(uniform.expand(y[full].shape))), "fully masked rows are not exactly 1 / sk"

    dy = _randn(b, np_, sq, sk, seed=sk + 1)
    ref.backward(dy.float())
    dy_buf = dy.clone()
    dx = sms.backward(dy_buf, y, scale)
    assert dx.data_ptr() == dy_buf.data_ptr()                                 # in place, like the reference
    assert torch.isfinite(dx[full].float()).all()
    _check_bwd(dx, dy, y, scale, f"masked softmax bwd sk={sk}")
    # autograd through masked_fill gives fully masked rows no gradient; the kernel (like the reference's) sees only y
    assert (dx.float() - xf.grad)[~full].abs().mean().item() <= 1e-3


def test_scaled_masked_softmax_rejects_sk_above_4096():
    x = torch.zeros(1, 1, 8, 4104, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="4096"):
        sms.forward(x, torch.zeros(1, 1, 8, 4104, dtype=torch.uint8, device="cuda"), 1.0)
    with pytest.raises(RuntimeError):
        sms.backward(x.clone(), x, 1.0)
    with pytest.raises(RuntimeError):
        suts.forward(torch.zeros(1, 4104, 4104, dtype=torch.bfloat16, device="cuda"), 1.0)


def test_get_batch_per_block_matches_reference_formula():
    # scaled_masked_softmax.h:337-349
    assert sms.get_batch_per_block(128, 2048, 2, 40) == 4
    assert sms.get_batch_per_block(128, 128, 2, 40) == 8
    assert sms.get_batch_per_block(128, 64, 2, 40) == 8
    assert sms.get_batch_per_block(128, 16, 2, 40) == 16


@pytest.mark.parametrize("ab,s", [(8, 64), (4, 512), (2, 2048), (3, 8), (2, 200), (2, 1000), (1, 4096)])
def test_scaled_upper_triang_masked_softmax(ab, s):
    x = _randn(ab, s, s, scale=2, seed=s)
    y = suts.forward(x, 0.25)
    causal = torch.triu(torch.ones(s, s, dtype=torch.bool, device="cuda"), 1)
    xf = x.float().requires_grad_(True)
    ref = torch.softmax((xf * 0.25).masked_fill(causal, float("-inf")), dim=-1)
    ref64 = torch.softmax((x.double() * 0.25).masked_fill(causal, float("-inf")), dim=-1)
    assert_ulp_close(y, ref64, f"causal softmax fwd s={s}", floor=1e-6)
    assert y.float().masked_select(causal).abs().max().item() == 0.0        # exact zeros above the diagonal
    dy = _randn(ab, s, s, seed=s + 1)
    ref.backward(dy.float())
    dy_buf = dy.clone()
    dx = suts.backward(dy_buf, y, 0.25)
    assert dx.data_ptr() == dy_buf.data_ptr()
    assert (dx.float() - xf.grad).abs().mean().item() <= 1e-3
    _check_bwd(dx, dy, y, 0.25, f"causal softmax bwd s={s}")
    assert dx.float().masked_select(causal).abs().max().item() == 0.0
