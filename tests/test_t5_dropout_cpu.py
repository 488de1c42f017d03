"""CPU: the mT5 dropout site table (fsb200/models/t5.py) against transformers' MT5 in training mode, and the decoder's
relative-position bias vector under the causal flag against HF's position bias plus causal mask."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200"))
import hf_oracle as H  # noqa: E402  (checker only)

from fsb200.models import t5_bias as TB  # noqa: E402


def site_table(Le, Ld, B, Se, Sd, d, nh, ff):
    """(site, kind, shape) of every dropout call of one training forward, in call order (the table of t5.py)."""
    hid = lambda S: ("hidden", (B, S, d))
    sites = [(0, *hid(Se))]
    for i in range(Le):
        sites += [(1 + 4 * i, "attn", (B, nh, Se, Se)), (2 + 4 * i, *hid(Se)), (3 + 4 * i, "hidden", (B, Se, ff)),
                  (4 + 4 * i, *hid(Se))]
    sites.append((1 + 4 * Le, *hid(Se)))
    E = 2 + 4 * Le
    sites.append((E, *hid(Sd)))
    for i in range(Ld):
        sites += [(E + 1 + 6 * i, "attn", (B, nh, Sd, Sd)), (E + 2 + 6 * i, *hid(Sd)), (E + 3 + 6 * i, "attn", (B, nh, Sd, Se)),
                  (E + 4 + 6 * i, *hid(Sd)), (E + 5 + 6 * i, "hidden", (B, Sd, ff)), (E + 6 + 6 * i, *hid(Sd))]
    sites.append((E + 1 + 6 * Ld, *hid(Sd)))
    return sites


def _hf(cfg, p):
    from transformers import MT5Config, MT5ForConditionalGeneration
    torch.manual_seed(0)
    config = MT5Config(dropout_rate=p, feed_forward_proj="gated-gelu", attn_implementation="eager", decoder_start_token_id=0,
                       pad_token_id=0, **cfg)
    return MT5ForConditionalGeneration(config).train()


@pytest.mark.parametrize("Le,Ld", [(3, 2), (1, 4)])
def test_dropout_calls_follow_the_site_table(Le, Ld, monkeypatch):
    cfg = dict(H.MT5_SMALL, num_layers=Le, num_decoder_layers=Ld)
    ref = _hf(cfg, 0.1)
    B, Se, Sd = 2, 24, 10
    batch = H.make_t5_batch(cfg["vocab_size"], B, Se, Sd, seed=3, pad_tail=5)
    calls = []
    real = torch.nn.functional.dropout

    def record(x, p=0.5, training=True, inplace=False):
        calls.append((tuple(x.shape), p, training))
        return real(x, p, training, inplace)

    monkeypatch.setattr(torch.nn.functional, "dropout", record)
    ref(**batch)
    want = site_table(Le, Ld, B, Se, Sd, cfg["d_model"], cfg["num_heads"], cfg["d_ff"])
    assert len(calls) == len(want) == 4 + 4 * Le + 6 * Ld
    assert [w[0] for w in want] == list(range(len(want)))
    for n, ((shape, p, training), (_, _, wshape)) in enumerate(zip(calls, want)):
        assert shape == wshape and p == 0.1 and training, (n, shape, wshape)


@pytest.mark.parametrize("S", [7, 40, 200])
def test_hf_decoder_bias_is_rel_bias_under_the_causal_flag(S):
    """HF's decoder self-attention adds position_bias + causal_mask to its scores: on and below the diagonal that is the
    bias vector as the kernels index it (offset k - q), above it a mask, which the causal flag applies."""
    ref = _hf(H.MT5_SMALL, 0.0)
    nh = H.MT5_SMALL["num_heads"]
    att = ref.decoder.block[0].layer[0].SelfAttention
    seen = {}

    def keep_bias(module, args, out):
        seen.setdefault("bias", out[1].detach())
    att.register_forward_hook(keep_bias)
    ids = torch.randint(2, H.MT5_SMALL["vocab_size"], (1, S))
    ref(input_ids=ids, labels=ids)
    hf_bias = seen["bias"][0]                                     # [heads, S, S]: position_bias + causal_mask
    rel = TB.rel_bias_vector(att.relative_attention_bias.weight.detach(), S, S, False, 32, 128)
    q = torch.arange(S)[:, None]
    k = torch.arange(S)[None, :]
    mine = rel[:, k - q + S - 1]                                  # [heads, S, S] as the kernels index it
    causal = (k <= q).expand(S, S)
    assert torch.equal(hf_bias[:, causal], mine[:, causal])
    assert (hf_bias[:, ~causal] <= torch.finfo(hf_bias.dtype).min / 2).all()
    scores = torch.randn(nh, S, S, generator=torch.Generator().manual_seed(S))
    want = torch.softmax(scores + hf_bias, -1)
    got = torch.softmax((scores + mine).masked_fill(~causal, float("-inf")), -1)
    assert torch.allclose(got, want, atol=1e-6, rtol=0)
    assert torch.equal(got.triu(1), torch.zeros_like(got))        # exactly zero above the diagonal
