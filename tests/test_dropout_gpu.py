"""GPU: dropout in the LayerNorm and standalone kernels and in BERT / MegatronBERT training (the attention dropout kernels
against fp64: tests/test_attention_dropout_gpu.py). Every mask is rebuilt by the numpy Philox of tests/philox_ref.py from the
layout documented in include/fsb200.h, never read from the library."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import philox_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)

from fsb200 import ops  # noqa: E402
from fsb200.models.bert import BertForMaskedLM, MegatronBertForPreTraining  # noqa: E402

DEV = "cuda"
SEED = 0x1234_5678_9ABC_DEF0


def _base(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


# ------------------------------------------------------------------------------------------------ op contract
def test_sdpa_dropout_rejects_bad_p_and_long_sequences():
    """p outside [0, 1) is refused when the Dropout is made; with p > 0 sequences are limited to 65536 (the attention mask
    layout of include/fsb200.h), the causal flag included."""
    with pytest.raises(RuntimeError, match="outside"):
        ops.Dropout(1.0, 1, _base(0), 0)
    k = torch.zeros(1, 65537, 1, 64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="65536"):
        ops.sdpa_fwd(k, k, k, 0.125, True, drop=ops.Dropout(0.1, 1, _base(0), 0))


def test_p_zero_entries_are_bit_identical_to_the_plain_ones():
    g = torch.Generator().manual_seed(0)
    d0 = ops.Dropout(0.0, 7, _base(0), 1)
    x = torch.randn(300, 768, generator=g).to(torch.bfloat16).to(DEV)
    r = torch.randn(300, 768, generator=g).to(torch.bfloat16).to(DEV)
    w = torch.randn(768, generator=g).to(torch.bfloat16).to(DEV)
    bb = torch.randn(768, generator=g).to(torch.bfloat16).to(DEV)
    y1, s1, x1 = ops.layernorm_fwd(x, w, bb, 1e-12, residual=r)
    y2, s2, x2 = ops.layernorm_fwd(x, w, bb, 1e-12, residual=r, drop=d0)
    assert torch.equal(y1, y2) and torch.equal(s1, s2) and torch.equal(x1, x2)
    dy = torch.randn(300, 768, generator=g).to(torch.bfloat16).to(DEV)
    gw1, gb1, gw2, gb2 = (torch.zeros(768, dtype=torch.float32, device=DEV) for _ in range(4))
    dx1 = ops.layernorm_bwd(dy, x1, w, s1, gw1, gb1, dres=r)
    dx2, dbr = ops.layernorm_bwd_dropout(dy, x1, w, s1, gw2, gb2, d0, dres=r)
    assert torch.equal(dx1, dx2) and torch.equal(dx1, dbr) and torch.equal(gw1, gw2) and torch.equal(gb1, gb2)


# ------------------------------------------------------------------------------------------------ LayerNorm / standalone
@pytest.mark.parametrize("rows,cols", [(300, 768), (64, 1024), (33, 2560)])
def test_layernorm_dropout_vs_fp64(rows, cols):
    p, site, base = 0.1, 5, _base(1 << 33)
    g = torch.Generator().manual_seed(cols)
    x = torch.randn(rows, cols, generator=g).to(torch.bfloat16).to(DEV)
    r = torch.randn(rows, cols, generator=g).to(torch.bfloat16).to(DEV)
    w = (1 + 0.1 * torch.randn(cols, generator=g)).to(torch.bfloat16).to(DEV)
    bb = (0.1 * torch.randn(cols, generator=g)).to(torch.bfloat16).to(DEV)
    drop = ops.Dropout(p, SEED, base, site)
    y, st, xs = ops.layernorm_fwd(x, w, bb, 1e-12, residual=r, drop=drop)
    keep = torch.from_numpy(R.hidden_keep(SEED, (1 << 33) + site, rows, cols, p)).to(DEV, torch.float64)
    xf = x.double().requires_grad_(True)
    sum_ref = xf * keep / (1 - p) + r.double()
    assert (xs.double() - sum_ref).abs().max().item() <= 2 ** -7 * sum_ref.abs().max().item()
    ref = torch.nn.functional.layer_norm(sum_ref, (cols,), w.double(), bb.double(), 1e-12)
    assert (y.double() - ref).abs().max().item() < 3e-2
    dy = torch.randn(rows, cols, generator=g).to(torch.bfloat16).to(DEV)
    dres = torch.randn(rows, cols, generator=g).to(torch.bfloat16).to(DEV)
    gw, gb = torch.zeros(cols, device=DEV), torch.zeros(cols, device=DEV)
    dx, dbr = ops.layernorm_bwd_dropout(dy, xs, w, st, gw, gb, drop, dres=dres)
    # reference backward from the kernel's own bf16 sum (the LN input), so only the LN backward and the mask are compared
    s_in = xs.double().requires_grad_(True)
    torch.nn.functional.layer_norm(s_in, (cols,), w.double(), bb.double(), 1e-12).backward(dy.double())
    dsum = s_in.grad + dres.double()
    for name, got, want in (("dx", dx, dsum), ("dbranch", dbr, dsum * keep / (1 - p))):
        err = (got.double() - want).abs().max().item()
        assert err < 2e-2 * max(1.0, want.abs().max().item()), f"{name}: {err}"


@pytest.mark.parametrize("rows,cols", [(257, 768), (10, 24)])
def test_standalone_dropout_vs_numpy_mask(rows, cols):
    p, site, base = 0.1, 0, _base(123)
    x = torch.randn(rows, cols, device=DEV).to(torch.bfloat16)
    drop = ops.Dropout(p, SEED, base, site)
    y = ops.dropout(x, drop)
    keep = torch.from_numpy(R.hidden_keep(SEED, 123, rows, cols, p)).to(DEV)
    keep_scale = np.float32(1.0) / (np.float32(1.0) - np.float32(p))     # the kernel's fp32 1 / (1 - p)
    want = torch.where(keep, x.float() * float(keep_scale), torch.zeros_like(x.float())).to(torch.bfloat16)
    assert torch.equal(y, want)


def test_drop_statistics():
    """>= 1e7 elements per site kind: the drop fraction is within 5 sigma of p_eff, two streams agree at the rate of two
    independent masks, and heads / rows / steps differ."""
    p = 0.1
    pe = R.p_eff(p)
    ones = torch.ones(4096, 2560, dtype=torch.bfloat16, device=DEV)
    base = _base(0)
    a = ops.dropout(ones, ops.Dropout(p, SEED, base, 0)) == 0
    b = ops.dropout(ones, ops.Dropout(p, SEED, base, 1)) == 0
    n = a.numel()
    sig = math.sqrt(pe * (1 - pe) / n)
    assert abs(a.float().mean().item() - pe) < 5 * sig
    agree = (a == b).float().mean().item()
    want = pe * pe + (1 - pe) ** 2
    assert abs(agree - want) < 5 * math.sqrt(want * (1 - want) / n)
    assert not torch.equal(a[0], a[1])
    # attention: V = identity rows recover P * Z / (1 - p) through the output; count zeros of P V with V one-hot
    B, Hh, S, D = 4, 8, 512, 64
    q = torch.zeros(B, S, Hh, D, dtype=torch.bfloat16, device=DEV)   # uniform P = 1 / S
    keep_counts = [torch.from_numpy(R.attn_keep(SEED, st, B, Hh, S, S, p)) for st in (0, 1)]
    ka = keep_counts[0]
    assert abs((~ka).float().mean().item() - pe) < 5 * math.sqrt(pe * (1 - pe) / ka.numel())
    assert not torch.equal(ka[0, 0], ka[0, 1])
    assert not torch.equal(keep_counts[0], keep_counts[1])
    # the kernel's drop fraction over >= 1e7 elements: with q = 0 and v = one-hot column of key k, O[.., d] = sum of kept P
    v = torch.zeros(B, S, Hh, D, dtype=torch.bfloat16, device=DEV)
    idx = torch.arange(S, device=DEV) % D
    v[:, torch.arange(S, device=DEV), :, idx] = 1.0
    dropped = 0
    total = 0
    for st in range(6):
        o, _ = ops.sdpa_fwd(q, q, v, 1.0, False, drop=ops.Dropout(p, SEED, _base(st), 0))
        want = torch.from_numpy(R.attn_keep(SEED, st, B, Hh, S, S, p)).to(DEV).float()
        onehot = torch.nn.functional.one_hot(idx, D).float()                 # [S, D]
        ref = torch.einsum("bhqk,kd->bqhd", want, onehot) / S / (1 - p)
        assert (o.float() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
        dropped += (1 - want).sum().item()
        total += want.numel()
    assert total >= 1e7
    assert abs(dropped / total - pe) < 5 * math.sqrt(pe * (1 - pe) / total)


# ------------------------------------------------------------------------------------------------ models
def _build_pair(cls_name, ph, pa, seed=0):
    from transformers import BertConfig, MegatronBertConfig
    import transformers
    cfgcls = BertConfig if cls_name == "bert" else MegatronBertConfig
    torch.manual_seed(seed)
    config = cfgcls(hidden_dropout_prob=ph, attention_probs_dropout_prob=pa, hidden_act="gelu", attn_implementation="eager",
                    **H.BERT_SMALL)
    ref = (transformers.BertForMaskedLM if cls_name == "bert" else transformers.MegatronBertForPreTraining)(config)
    ref.train()
    H._bf16_exact_(ref)
    mine = (BertForMaskedLM if cls_name == "bert" else MegatronBertForPreTraining)(config, device="cuda")
    mine.load_reference_state_dict(ref.state_dict())
    return ref, mine


@pytest.mark.parametrize("cls_name", ["bert", "megatron"])
def test_model_parity_with_replayed_masks(cls_name, monkeypatch):
    ph, pa = 0.1, 0.2
    ref, mine = _build_pair(cls_name, ph, pa)
    nsp = cls_name == "megatron"
    batch = H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 3, 96, seed=5, nsp=nsp, pad_tail=20)
    B, S = batch["input_ids"].shape
    h, nh, nl = H.BERT_SMALL["hidden_size"], H.BERT_SMALL["num_attention_heads"], H.BERT_SMALL["num_hidden_layers"]
    seed = mine.dropout_seed
    assert int(mine.dropout_counter.item()) == 0
    sites = [("hidden", 0)]
    for i in range(nl):
        sites += [("attn", 1 + 3 * i), ("hidden", 2 + 3 * i), ("hidden", 3 + 3 * i)]
    calls = []

    def replay(x, p=0.5, training=True, inplace=False):
        kind, site = sites[len(calls)]
        if kind == "hidden":
            assert tuple(x.shape) == (B, S, h) and p == ph
            keep = R.hidden_keep(seed, site, B * S, h, p).reshape(B, S, h)
        else:
            assert tuple(x.shape) == (B, nh, S, S) and p == pa
            keep = R.attn_keep(seed, site, B, nh, S, S, p)
        calls.append(site)
        return x * torch.from_numpy(keep).to(x.dtype) / (1.0 - p)

    monkeypatch.setattr(torch.nn.functional, "dropout", replay)
    out_ref = ref(**batch)
    assert len(calls) == len(sites) == mine.dropout_sites
    out_ref.loss.backward()
    monkeypatch.undo()
    out = mine(**{k: v.cuda() for k, v in batch.items()}, return_logits=True)
    assert int(mine.dropout_counter.item()) == mine.dropout_sites
    assert abs(out.loss.item() - out_ref.loss.item()) <= 4e-3, (out.loss.item(), out_ref.loss.item())
    ref_logits = out_ref.logits if getattr(out_ref, "logits", None) is not None else out_ref.prediction_logits
    assert (out.logits.float().cpu() - ref_logits.detach()).abs().max().item() <= 4 * 2.0 ** -8 * ref_logits.abs().max().item()
    out.loss.backward()
    torch.cuda.synchronize()
    refp = dict(ref.named_parameters())
    for name, prm in mine.named_parameters():
        want = refp[name].grad
        got = prm.main_grad.float().cpu()
        if want is None or want.norm().item() < 1e-7:
            assert got.norm().item() < 1e-4, name
            continue
        cos = torch.dot(got.flatten(), want.flatten()) / (got.norm() * want.norm() + 1e-30)
        assert cos.item() >= 0.998, (name, cos.item())
        assert abs(got.norm().item() / want.norm().item() - 1.0) <= 0.03, (name, got.norm().item(), want.norm().item())


def _grads(cls_name, torch_seed, batch):
    torch.manual_seed(torch_seed)
    _, mine = _build_pair(cls_name, 0.1, 0.1)
    torch.manual_seed(torch_seed)   # the dropout seed is drawn at construction
    cls = BertForMaskedLM if cls_name == "bert" else MegatronBertForPreTraining
    m2 = cls(mine.config, device="cuda")
    m2.load_reference_state_dict({k: v.data for k, v in mine._p.items()})
    out = m2(**{k: v.cuda() for k, v in batch.items()})
    out.loss.backward()
    torch.cuda.synchronize()
    return out.loss.item(), torch.cat([p.main_grad.flatten().float() for p in m2._p.values()])


def test_determinism_and_seed_dependence():
    batch = H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 2, 64, seed=9, nsp=True)
    l1, g1 = _grads("megatron", 17, batch)
    l2, g2 = _grads("megatron", 17, batch)
    l3, g3 = _grads("megatron", 18, batch)
    assert l1 == l2 and torch.equal(g1, g2)
    assert l1 != l3 and not torch.equal(g1, g3)


@pytest.mark.parametrize("cls_name", ["bert", "megatron"])
def test_eval_mode_equals_dropout_free_config_and_train_mode_no_grad_drops(cls_name):
    ref, mine = _build_pair(cls_name, 0.1, 0.1)
    _, plain = _build_pair(cls_name, 0.0, 0.0)
    plain.load_reference_state_dict(ref.state_dict())
    batch = {k: v.cuda() for k, v in H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 2, 64, seed=4, nsp=cls_name == "megatron",
                                                      pad_tail=7).items()}
    mine.eval()
    with torch.no_grad():
        a = mine(**batch, return_logits=True)
        b = plain(**batch, return_logits=True)
    assert torch.equal(a.logits, b.logits) and a.loss.item() == b.loss.item()
    assert int(mine.dropout_counter.item()) == 0             # eval draws no masks
    mine.train()
    with torch.no_grad():
        c = mine(**batch, return_logits=True)
    assert not torch.equal(c.logits, b.logits)
    assert int(mine.dropout_counter.item()) == mine.dropout_sites


def _graph_vs_eager(stage, ga, p):
    """Five PretrainStep steps of a MegatronBERT, eager and as a replayed CUDA graph: (losses, params, counter) of each."""
    from fsb200.trainer import PretrainStep
    runs = []
    for graph in (False, True):
        torch.manual_seed(3)
        _, model = _build_pair("megatron", p, p)
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, weight_decay=0.01, grad_clip=1.0, ga_steps=ga, stage=stage,
                          cuda_graph=graph)
        losses = []
        for it in range(5):
            # no attention_mask: the forward reads whether a padding mask is needed on the host, which a capture cannot do
            mbs = [{k: v.cuda() for k, v in H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 2, 64, seed=50 + 2 * it + m,
                                                             nsp=True).items() if k != "attention_mask"} for m in range(ga)]
            losses.append(float(st.step_device(mbs)))
        counter = None if model.dropout_counter is None else int(model.dropout_counter.item())
        runs.append((losses, model.flat.params.clone(), counter, model.dropout_sites))
    return runs


# ZeRO-2 with GA 2, which accumulates each bucket as soon as its backward finishes, is checked below, with and without dropout.
@pytest.mark.parametrize("stage,ga", [(1, 1), (2, 1), (1, 2)])
def test_cuda_graph_step_equals_eager_with_dropout(stage, ga):
    (l0, p0, c0, sites), (l1, p1, c1, _) = _graph_vs_eager(stage, ga, 0.1)
    assert c0 == c1 == 5 * ga * sites
    assert max(abs(a - b) for a, b in zip(l0, l1)) < 1e-5, (l0, l1)
    assert torch.equal(p0, p1), (p0.float() - p1.float()).abs().max()


# The final encoder LayerNorm's weight gradient lives in the head bucket, so that bucket is reported only after the LN backward.
# Reported before it, ZeRO-2 with GA 2 accumulated the previous micro-batch's value, which differs between a first eager step
# (zeros) and a first replay (what the capture passes left).
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_cuda_graph_step_equals_eager_zero2_ga2(p):
    (l0, p0, _, _), (l1, p1, _, _) = _graph_vs_eager(2, 2, p)
    assert l0 == l1, (l0, l1)
    assert torch.equal(p0, p1), (p0.float() - p1.float()).abs().max()


def test_micro_batches_of_one_step_get_different_masks():
    torch.manual_seed(3)
    _, model = _build_pair("bert", 0.1, 0.1)
    b = {k: v.cuda() for k, v in H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 2, 64, seed=1).items()}
    with torch.no_grad():
        l1 = model(**b, return_logits=True).logits.clone()
        l2 = model(**b, return_logits=True).logits.clone()
    assert not torch.equal(l1, l2)
