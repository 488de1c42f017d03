"""CPU checks for FP8 training of BERT / MegatronBERT: the FP8 GEMM verifier with the bias / GELU / aux epilogue
(tests/fp8_epilogue_refs.py) rejects the faults such an epilogue can make (a lost bias, the other GELU form, aux holding the post-activation,
a lost accumulate term, an uninverted scale), Fp8Linear's construction rules, and the example's --fp8 flag."""
import os
import sys

import pytest
import torch

import fp8_epilogue_refs as E
import fp8_ref
import launch_refs as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F32 = torch.bfloat16, torch.float32


def _ok(fn, *args, **kw):
    b = R.Bound("cpu")
    fn(b, *args, **kw)
    assert b.worst <= 1.0


def _rejects(fn, *args, **kw):
    with pytest.raises(AssertionError):
        fn(R.Bound("cpu"), *args, **kw)


def _operands(m=96, n=80, k=32):
    """e4m3 codes of A [m, k] and W [n, k] with their scales, a bias whose pre-activations reach well into x < -2 (where
    the erf and tanh GELU differ by up to 4e-4, many bf16 ulps), and an old D. The products are small next to the bias, so
    the FP8 accumulation bound (2^-9 sum |A||B| ~ 1e-4 here) stays below that difference."""
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(m, k, generator=g) * 0.05).to(BF16)
    w = (torch.randn(n, k, generator=g) * 0.05).to(BF16)
    aq, _, sa = fp8_ref.quantize(x.float().numpy(), "e4m3")
    wq, _, sw = fp8_ref.quantize(w.float().numpy(), "e4m3")
    A, W = torch.from_numpy(aq).view(torch.float8_e4m3fn), torch.from_numpy(wq).view(torch.float8_e4m3fn)
    SA, SW = torch.tensor([sa], dtype=F32), torch.tensor([sw], dtype=F32)
    bias = (torch.randn(n, generator=g) * 2.0 - 1.0).to(BF16)
    old = torch.randn(m, n, generator=g).to(BF16)
    prod = (A.float().double() * SA.double()) @ (W.float().double() * SW.double()).t()
    return A, SA, W, SW, bias, old, prod


@pytest.mark.parametrize("epi", [R.EPI_GELU_TANH, R.EPI_GELU_ERF])
@pytest.mark.parametrize("accumulate", [False, True])
def test_fp8_epilogue_verifier_accepts_the_right_answer_and_rejects_faults(epi, accumulate):
    A, SA, W, SW, bias, old, prod = _operands()
    act = R._EPI_ACT[epi]
    other = R.ACT_GELU_ERF if act == R.ACT_GELU_TANH else R.ACT_GELU_TANH
    o = old.double() if accumulate else 0.0
    oldarg = old if accumulate else None
    pre = prod + bias.double()
    aux = pre.to(BF16)
    d = (R.act64(act, pre) + o).to(BF16)
    assert (pre < -2).sum() > 100                     # the construction reaches where the two GELU forms differ
    _ok(E.verify_gemm_fp8, A, SA, W, SW, d, oldarg, bias=bias, epilogue=epi, aux=aux)
    # a lost bias (in D, and in aux alone)
    _rejects(E.verify_gemm_fp8, A, SA, W, SW, (R.act64(act, prod) + o).to(BF16), oldarg, bias=bias, epilogue=epi, aux=aux)
    _rejects(E.verify_gemm_fp8, A, SA, W, SW, d, oldarg, bias=bias, epilogue=epi, aux=prod.to(BF16))
    # the other GELU form
    _rejects(E.verify_gemm_fp8, A, SA, W, SW, (R.act64(other, pre) + o).to(BF16), oldarg, bias=bias, epilogue=epi, aux=aux)
    # aux holding the post-activation
    _rejects(E.verify_gemm_fp8, A, SA, W, SW, d, oldarg, bias=bias, epilogue=epi, aux=R.act64(act, pre).to(BF16))
    # an uninverted scale
    un = (A.float().double() / SA.double()) @ (W.float().double() * SW.double()).t() + bias.double()
    _rejects(E.verify_gemm_fp8, A, SA, W, SW, (R.act64(act, un) + o).to(BF16), oldarg, bias=bias, epilogue=epi,
             aux=un.to(BF16))
    if accumulate:   # the accumulate term lost
        _rejects(E.verify_gemm_fp8, A, SA, W, SW, R.act64(act, pre).to(BF16), old, bias=bias, epilogue=epi, aux=aux)


def test_fp8_bias_only_verifier():
    """Bias without activation (the q|k|v, attention-output and output projections): D = pre, and a lost bias fails."""
    A, SA, W, SW, bias, _, prod = _operands()
    pre = prod + bias.double()
    _ok(E.verify_gemm_fp8, A, SA, W, SW, pre.to(BF16), None, bias=bias)
    _rejects(E.verify_gemm_fp8, A, SA, W, SW, prod.to(BF16), None, bias=bias)
    _ok(E.verify_gemm_fp8, A, SA, W, SW, prod.to(BF16))   # the plain path is unchanged


def test_fp8linear_takes_a_bias_and_refuses_conv1d():
    from fsb200.models.layers import Fp8Linear, Linear
    w, b = torch.zeros(32, 16, dtype=BF16), torch.zeros(32, dtype=BF16)
    gw, gb = torch.zeros_like(w), torch.zeros_like(b)
    f = Fp8Linear(Linear(w, gw, b, gb))
    assert f.bias_grad is gb and f.lin.bias is b
    with pytest.raises(ValueError, match="Conv1D"):
        Fp8Linear(Linear(w, gw, b, gb, conv1d=True))


def test_example_fp8_flag_parses(tmp_path):
    import runpy
    import hf_fixtures as F
    import hf_recipes
    for p in ("fengshen-lm_b200", os.path.join("fengshen-lm_b200", "compat")):
        if os.path.join(ROOT, p) not in sys.path:
            sys.path.insert(0, os.path.join(ROOT, p))
    F.bert_dir(tmp_path / "m")
    corpus = F.bert_corpus(tmp_path / "train.json", n=8)
    ns = runpy.run_path(hf_recipes.EXAMPLE, run_name="example_not_main")
    base = ["--model_path", str(tmp_path / "m"), "--train_file", str(corpus)]
    assert ns["parse_args"](base).fp8 is False
    assert ns["parse_args"](base + ["--fp8"]).fp8 is True
