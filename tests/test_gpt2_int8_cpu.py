"""The fp64 references of the W8A16 / W4A16 bias / GELU epilogue (tests/wq_epilogue_refs.py, which the int8 / int4 GPT-2
tests and launch census rely on) held to an independent torch
computation: the right answer passes, the answers of the likely bugs do not."""
import pytest
import torch
import torch.nn.functional as F

import int4_ref
import int8_ref
import launch_refs as R
import wq_epilogue_refs as E

BF16 = torch.bfloat16


def _randn(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF16)


def _ok(fn, *args, **kw):
    b = R.Bound("cpu")
    fn(b, *args, **kw)
    assert b.worst <= 1.0


def _rejects(fn, *args, **kw):
    with pytest.raises(AssertionError):
        fn(R.Bound("cpu"), *args, **kw)


def _operands(fmt, n=64, k=384, m=24):
    w = _randn(n, k, seed=1, scale=0.05)
    if fmt == "int8":
        qn, sn = int8_ref.quantize(w.float().numpy())
        q, s = torch.from_numpy(qn), torch.from_numpy(sn)
        W = q.double() * s.double()[:, None]
        verify = E.verify_gemm_w8a16
    else:
        qn, sn = int4_ref.quantize(w.float().numpy())
        q, s = torch.from_numpy(int4_ref.pack(qn)), torch.from_numpy(sn).to(BF16)
        W = torch.from_numpy(int4_ref.dequantize(qn, sn)).double()
        verify = E.verify_gemm_w4a16
    return _randn(m, k, seed=2), q, s, W, _randn(n, seed=3, scale=0.5), verify


@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_bias_epilogue_reference_against_torch(fmt):
    a, q, s, W, bias, verify = _operands(fmt)
    pre = a.double() @ W.t() + bias.double()
    for epi, act in ((R.EPI_NONE, lambda x: x), (R.EPI_GELU_TANH, lambda x: F.gelu(x, approximate="tanh"))):
        out = act(pre).to(BF16)
        _ok(verify, a, q, s, out, bias, epi)
        _rejects(verify, a, q, s, act(pre + bias.double()).to(BF16), bias, epi)         # bias added twice (once per split)
        _rejects(verify, a, q, s, act(a.double() @ W.t()).to(BF16), bias, epi)          # bias lost
        _rejects(verify, a, q, s, act(pre + 0.25 * bias.double().roll(1)).to(BF16), bias, epi)   # a neighbour's bias
    _rejects(verify, a, q, s, pre.to(BF16), bias, R.EPI_GELU_TANH)                       # GELU not applied
    _rejects(verify, a, q, s, F.gelu(pre).to(BF16) * 1.01, bias, R.EPI_GELU_TANH)
    # without a bias the reference is the one the bias-free GEMM is held to
    _ok(verify, a, q, s, (a.double() @ W.t()).to(BF16))


def test_int8_bias_reference_rejects_scale_after_bias():
    """int8 scales the sum before the bias is added: s (acc + bias) is a different answer."""
    a, q, s, _, bias, verify = _operands("int8")
    acc = a.double() @ q.double().t()
    wrong = (s.double() * (acc + bias.double())).to(BF16)
    _rejects(verify, a, q, s, wrong, bias, R.EPI_NONE)
    _ok(verify, a, q, s, (s.double() * acc + bias.double()).to(BF16), bias, R.EPI_NONE)
