"""CPU: the GPT-2 dropout site table (fsb200/models/gpt2.py) against transformers' GPT2LMHeadModel in training mode, and the
launch checkers of tests/launch_refs.py on causal + padding + dropout attention, the form GPT-2's attention takes."""
import math
import os
import sys

import pytest
import torch

import launch_refs as R
import philox_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)

BF16 = torch.bfloat16


def site_table(L, B, S, h, nh, pe, pa, pr):
    """(site, kind, shape, p) of every dropout call of one training forward, in call order (the table of gpt2.py). Sites whose
    probability is 0 are listed too: transformers calls F.dropout there as well."""
    sites = [(0, "hidden", (B, S, h), pe)]
    for i in range(L):
        sites += [(1 + 3 * i, "attn", (B, nh, S, S), pa), (2 + 3 * i, "hidden", (B, S, h), pr),
                  (3 + 3 * i, "hidden", (B, S, h), pr)]
    return sites


def hf_gpt2(cfg, pe, pa, pr, seed=0):
    from transformers import GPT2Config, GPT2LMHeadModel
    torch.manual_seed(seed)
    config = GPT2Config(embd_pdrop=pe, attn_pdrop=pa, resid_pdrop=pr, activation_function="gelu_new",
                        attn_implementation="eager", **cfg)
    return GPT2LMHeadModel(config).train()


@pytest.mark.parametrize("L", [2, 3])
@pytest.mark.parametrize("probs", [(0.1, 0.2, 0.05), (0.1, 0.0, 0.1)], ids=["distinct", "attn0"])
def test_dropout_calls_follow_the_site_table(L, probs, monkeypatch):
    cfg = dict(H.GPT2_SMALL, n_layer=L)
    ref = hf_gpt2(cfg, *probs)
    B, S = 2, 24
    batch = H.make_lm_batch(cfg["vocab_size"], B, S, seed=3)
    batch["attention_mask"][1, S - 5:] = 0
    calls = []
    real = torch.nn.functional.dropout

    def record(x, p=0.5, training=True, inplace=False):
        calls.append((tuple(x.shape), p, training))
        return real(x, p, training, inplace)

    monkeypatch.setattr(torch.nn.functional, "dropout", record)
    ref(**batch)
    want = site_table(L, B, S, cfg["n_embd"], cfg["n_head"], *probs)
    assert len(calls) == len(want) == 1 + 3 * L
    assert [w[0] for w in want] == list(range(len(want)))
    for n, ((shape, p, training), (_, _, wshape, wp)) in enumerate(zip(calls, want)):
        assert shape == wshape and p == wp and training, (n, shape, wshape, p, wp)


# ------------------------------------------------------------------------------------------------ causal + dropout checkers
def _randn(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(BF16)


def _causal_dropout_autograd(q, k, v, scale, kvm, dout, m, causal=True):
    S = q.shape[1]
    qd, kd, vd = (R._bhsd(t).double().requires_grad_(True) for t in (q, k, v))
    s = scale * qd @ kd.transpose(-1, -2)
    if causal:
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
    s = s.masked_fill((kvm == 0)[:, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = (torch.softmax(s, -1) * m) @ vd
    o.backward(R._bhsd(dout).double())
    return o.detach(), lse.detach(), (qd.grad, kd.grad, vd.grad)


def test_causal_sdpa_dropout_checkers():
    """verify_sdpa_fwd / verify_sdpa_bwd with causal=True, a right-padding kv_mask and a DropSpec accept the exact answer and
    reject the mask of site + 1, a mask transposed in (q, k), a mask without its 1 / (1 - p), a stream that lost its high
    word, and an attention that ignores the causal mask."""
    B, S, H, D = 2, 80, 2, 64
    q, k, v, dout = (_randn(B, S, H, D, seed=s) for s in (1, 2, 3, 9))
    kvm = torch.ones(B, S, dtype=torch.uint8)
    kvm[1, 61:] = 0
    scale = 1.0 / math.sqrt(D)
    d = R.DropSpec(0.1, 0x1234_5678_9ABC_DEF, 2 ** 32 + 2)

    def mask(dd, scaled=True, transpose=False):
        z = philox_ref.attn_keep_t(dd.seed, dd.stream, range(B), H, S, S, dd.p).double()
        z = z.transpose(-1, -2) if transpose else z
        return z * R.keep_scale(dd.p) if scaled else z
    o, lse, (dq, dk, dv) = _causal_dropout_autograd(q, k, v, scale, kvm, dout, mask(d))
    O, L2 = R._bhsd(o).to(BF16), (lse / math.log(2.0)).float()
    fa = (q, k, v, scale, True, kvm, None)
    R_ok = R.Bound("cpu")
    R.verify_sdpa_fwd(R_ok, *fa, O, L2, d)
    ba = (q, k, v, O, dout, L2, scale, True)
    DQ, DK, DV = (R._bhsd(t).to(BF16) for t in (dq, dk, dv))
    R.verify_sdpa_bwd(R_ok, *ba, DQ, DK, DV, kvm, None, None, None, d)
    assert R_ok.worst <= 1.0
    faults = {"site + 1": mask(d._replace(stream=d.stream + 1)), "transposed (q, k)": mask(d, transpose=True),
              "no 1 / (1 - p)": mask(d, scaled=False), "high word lost": mask(d._replace(stream=d.stream & 0xFFFFFFFF))}
    for name, m in faults.items():
        o_, _, (_, _, dv_) = _causal_dropout_autograd(q, k, v, scale, kvm, dout, m)
        with pytest.raises(AssertionError):
            R.verify_sdpa_fwd(R.Bound("cpu"), *fa, R._bhsd(o_).to(BF16), L2, d)
        with pytest.raises(AssertionError):   # fed the right forward's O: dV alone already differs
            R.verify_sdpa_bwd(R.Bound("cpu"), *ba, DQ, DK, R._bhsd(dv_).to(BF16), kvm, None, None, None, d)
    o_, lse_, _ = _causal_dropout_autograd(q, k, v, scale, kvm, dout, mask(d), causal=False)
    with pytest.raises(AssertionError):
        R.verify_sdpa_fwd(R.Bound("cpu"), *fa, R._bhsd(o_).to(BF16), (lse_ / math.log(2.0)).float(), d)
