"""GPU: attention with dropout on its probabilities against fp64, in every form the models launch it: BERT / MegatronBERT
(with and without padding), mT5's encoder (relative bias + padding) and decoder (causal flag + relative bias), GPT-2 (causal
flag, with and without padding). Every mask is rebuilt by the numpy Philox of tests/philox_ref.py from the layout
documented in include/fsb200.h, never read from the library."""
import math
from collections import namedtuple

import pytest
import torch

import philox_ref as R

from fsb200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"

# causal flag, relative bias, padded key ranges (row, start, end) at length S, the lengths, and the Philox seed, stream base
# and site. S = 200 ends inside a query / key tile; the bases 2^33 and 2^32 + 3 put the stream in the high word.
Form = namedtuple("Form", "causal bias padding seqs seed base site")
_BERT = dict(seqs=(128, 200, 512), seed=0x1234_5678_9ABC_DEF0, base=11, site=3)
_T5 = dict(seqs=(128, 200, 512), seed=0x0FED_CBA9_8765_4321, base=1 << 33, site=4)
_GPT2 = dict(seqs=(128, 200, 1024), seed=0x2468_ACE0_1357_9BDF, base=(1 << 32) + 3, site=4)
FORMS = {
    "bert": Form(False, False, lambda S: (), **_BERT),
    "bert_padding": Form(False, False, lambda S: ((0, S - 37, S), (1, 5, 21)), **_BERT),
    "t5_encoder": Form(False, True, lambda S: ((1, S - 29, S),), **_T5),
    "t5_decoder": Form(True, True, lambda S: (), **_T5),
    "gpt2": Form(True, False, lambda S: (), **_GPT2),
    # right padding, as a padded fine-tuning batch has it; row 1 ends inside a 128-row tile
    "gpt2_padding": Form(True, False, lambda S: ((1, S - 37, S),), **_GPT2),
}
CASES = [(name, S) for name, f in FORMS.items() for S in f.seqs]


def _base(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _case(f, D, S, seed):
    B, Hh = 2, 2
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, S, 3, Hh, D, generator=g).to(torch.bfloat16).to(DEV)
    rel = torch.randn(Hh, 2 * S - 1, generator=g).to(DEV) if f.bias else None
    mask = None
    if f.padding(S):
        mask = torch.ones(B, S, dtype=torch.uint8, device=DEV)
        for row, lo, hi in f.padding(S):
            mask[row, lo:hi] = 0
    dout = torch.randn(B, S, Hh, D, generator=g).to(torch.bfloat16).to(DEV)
    return qkv, rel, mask, dout


def _run(f, qkv, rel, mask, dout, scale, drop):
    """Forward + backward -> (out, lse, dqkv, drel or None)."""
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    out, lse = ops.sdpa_fwd(q, k, v, scale, f.causal, kv_mask=mask, rel_bias=rel, drop=drop)
    dqkv = torch.full_like(qkv, float("nan"))
    drel = None if rel is None else torch.zeros_like(rel)
    ops.sdpa_bwd(q, k, v, out, dout, lse, scale, f.causal, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], kv_mask=mask,
                 rel_bias=rel, drel_bias=drel, drop=drop)
    return out, lse, dqkv, drel


def _same(a, b):
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("form,S", CASES, ids=[f"{n}-{S}" for n, S in CASES])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_attention_dropout_vs_fp64(form, S, D, p):
    """The diagonal tiles of a causal form are where the causal mask and the drop bits meet, in the forward's two consumer
    warpgroups and the dK / dV kernel's transposed fragment."""
    f = FORMS[form]
    B, Hh = 2, 2
    qkv, rel, mask, dout = _case(f, D, S, S + D)
    scale = 1.0 / math.sqrt(D)
    drop = ops.Dropout(p, f.seed, _base(f.base), f.site)
    out, lse, dqkv, drel = _run(f, qkv, rel, mask, dout, scale, drop)
    torch.cuda.synchronize()
    keep = torch.from_numpy(R.attn_keep(f.seed, f.base + f.site, B, Hh, S, S, p)).to(DEV, torch.float64)
    qf, kf, vf = (qkv[:, :, i].double().detach().requires_grad_(True) for i in range(3))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    if rel is not None:
        relf = rel.double().detach().requires_grad_(True)
        i = torch.arange(S, device=DEV)
        s = s + relf[:, i[None, :] - i[:, None] + S - 1][None]
    if f.causal:
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=DEV).tril(), float("-inf"))
    if mask is not None:
        s = s.masked_fill(~mask.bool()[:, None, None, :], float("-inf"))
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1) * keep / (1.0 - p), vf)
    assert not torch.isnan(out.float()).any() and not torch.isnan(lse).any()
    assert (out.double() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item() / 4)
    assert (lse.double() * math.log(2.0) - torch.logsumexp(s, -1)).abs().max().item() < 2e-3
    ref.backward(dout.double())
    grads = [("dq", dqkv[:, :, 0], qf.grad), ("dk", dqkv[:, :, 1], kf.grad), ("dv", dqkv[:, :, 2], vf.grad)]
    if rel is not None:
        grads.append(("drel", drel, relf.grad))
    for name, got, want in grads:
        assert not torch.isnan(got.float()).any(), name
        err = (got.double() - want).abs().max().item()
        assert err < 3e-2 * max(1.0, want.abs().max().item()), f"{name}: {err}"
    if f.causal and rel is not None:
        assert torch.equal(drel[:, S:], torch.zeros_like(drel[:, S:]))   # masked offsets k - q > 0 get no gradient
    assert _same((out, lse, dqkv, drel), _run(f, qkv, rel, mask, dout, scale, drop))   # deterministic


def test_p_zero_is_bit_identical_to_no_dropout():
    d0 = ops.Dropout(0.0, 7, _base(0), 1)
    for name, f in FORMS.items():
        qkv, rel, mask, dout = _case(f, 64, 200, 1)
        a = _run(f, qkv, rel, mask, dout, 0.125, None)
        b = _run(f, qkv, rel, mask, dout, 0.125, d0)
        assert _same(a, b), name
