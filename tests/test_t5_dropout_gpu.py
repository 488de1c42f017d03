"""GPU: mT5 dropout — the RMSNorm and gated-activation dropout kernels, and the model against transformers' MT5 on replayed
masks (its attention forms against fp64: tests/test_attention_dropout_gpu.py). Every mask is rebuilt by the numpy Philox of
tests/philox_ref.py from the layout documented in include/fsb200.h, never read from the library."""
import copy
import math
import os
import sys

import pytest
import torch

import philox_ref as R
from test_t5_dropout_cpu import site_table

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)

from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.models.t5 import MT5ForConditionalGeneration  # noqa: E402

DEV = "cuda"
SEED = 0x0FED_CBA9_8765_4321


def _base(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


# ------------------------------------------------------------------------------------------------ p = 0
def test_p_zero_entries_are_bit_identical_to_the_plain_ones():
    d0 = ops.Dropout(0.0, 7, _base(0), 1)
    g = torch.Generator().manual_seed(2)
    x, r, dy, dres = (torch.randn(300, 1024, generator=g).to(torch.bfloat16).to(DEV) for _ in range(4))
    w = torch.randn(1024, generator=g).to(torch.bfloat16).to(DEV)
    y1, s1, x1 = ops.rmsnorm_fwd(x, w, 1e-6, residual=r)
    y2, s2, x2 = ops.rmsnorm_fwd(x, w, 1e-6, residual=r, drop=d0)
    assert torch.equal(y1, y2) and torch.equal(s1, s2) and torch.equal(x1, x2)
    gw1, gw2 = torch.zeros(1024, device=DEV), torch.zeros(1024, device=DEV)
    dx1 = ops.rmsnorm_bwd(dy, x1, w, s1, gw1, dres=dres)
    dx2, dbr = ops.rmsnorm_bwd_dropout(dy, x1, w, s1, gw2, d0, dres=dres)
    assert torch.equal(dx1, dx2) and torch.equal(dx1, dbr) and torch.equal(gw1, gw2)
    gu = torch.randn(300, 2 * 1032, generator=g).to(torch.bfloat16).to(DEV)
    a1 = ops.glu_fwd(L.ACT_GELU_TANH, gu[:, :1032], gu[:, 1032:])
    a2 = ops.glu_fwd(L.ACT_GELU_TANH, gu[:, :1032], gu[:, 1032:], drop=d0)
    assert torch.equal(a1, a2)
    da = torch.randn(300, 1032, generator=g).to(torch.bfloat16).to(DEV)
    g1, g2 = torch.empty_like(gu), torch.empty_like(gu)
    ops.glu_bwd(L.ACT_GELU_TANH, da, gu[:, :1032], gu[:, 1032:], g1[:, :1032], g1[:, 1032:])
    ops.glu_bwd(L.ACT_GELU_TANH, da, gu[:, :1032], gu[:, 1032:], g2[:, :1032], g2[:, 1032:], drop=d0)
    assert torch.equal(g1, g2)


# ------------------------------------------------------------------------------------------------ RMSNorm / gated activation
@pytest.mark.parametrize("rows,cols", [(333, 1024), (77, 2816)])
def test_rmsnorm_dropout_vs_fp64(rows, cols):
    p, site, base = 0.1, 9, _base(5)
    g = torch.Generator().manual_seed(cols)
    x, r, dy, dres = (torch.randn(rows, cols, generator=g).to(torch.bfloat16).to(DEV) for _ in range(4))
    w = (1 + 0.1 * torch.randn(cols, generator=g)).to(torch.bfloat16).to(DEV)
    drop = ops.Dropout(p, SEED, base, site)
    y, rstd, xs = ops.rmsnorm_fwd(x, w, 1e-6, residual=r, drop=drop)
    keep = torch.from_numpy(R.hidden_keep(SEED, 5 + site, rows, cols, p)).to(DEV, torch.float64)
    sum_ref = x.double() * keep / (1 - p) + r.double()
    assert (xs.double() - sum_ref).abs().max().item() <= 2 ** -7 * sum_ref.abs().max().item()
    rms = lambda t: t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6)
    y_ref = rms(xs.double()) * w.double()
    assert (y.double() - y_ref).abs().max().item() < 2e-2 * y_ref.abs().max().item()
    gw = torch.full((cols,), float("nan"), device=DEV)
    dx, dbr = ops.rmsnorm_bwd_dropout(dy, xs, w, rstd, gw, drop, dres=dres)
    s_in = xs.double().requires_grad_(True)
    wf = w.double().requires_grad_(True)
    (rms(s_in) * wf).backward(dy.double())      # from the kernel's own bf16 sum: only the backward and the mask are compared
    dsum = s_in.grad + dres.double()
    for name, got, want in (("dx", dx, dsum), ("dbranch", dbr, dsum * keep / (1 - p)), ("dscale", gw, wf.grad)):
        err = (got.double() - want).abs().max().item()
        assert err < 2e-2 * max(1.0, want.abs().max().item()), f"{name}: {err}"


def _gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x.pow(3))))


@pytest.mark.parametrize("rows,ff", [(333, 2816), (61, 1032)])     # 1032: a multiple of 8, not of 16
def test_glu_dropout_vs_fp64(rows, ff):
    p, site, base = 0.1, 2, _base(77)
    g = torch.Generator().manual_seed(ff)
    gu = torch.randn(rows, 2 * ff, generator=g).to(torch.bfloat16).to(DEV)      # [T, 2 ff]: the wi_0 | wi_1 GEMM output
    drop = ops.Dropout(p, SEED, base, site)
    out = ops.glu_fwd(L.ACT_GELU_TANH, gu[:, :ff], gu[:, ff:], drop=drop)
    keep = torch.from_numpy(R.hidden_keep(SEED, 77 + site, rows, ff, p)).to(DEV, torch.float64)
    gf, uf = (t.double().requires_grad_(True) for t in (gu[:, :ff], gu[:, ff:]))
    ref = _gelu_tanh(gf) * uf * keep / (1 - p)
    assert (out.double() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    assert torch.equal(out[keep == 0], torch.zeros_like(out[keep == 0]))
    dout = torch.randn(rows, ff, generator=g).to(torch.bfloat16).to(DEV)
    dgu = torch.full_like(gu, float("nan"))
    ops.glu_bwd(L.ACT_GELU_TANH, dout, gu[:, :ff], gu[:, ff:], dgu[:, :ff], dgu[:, ff:], drop=drop)
    ref.backward(dout.double())
    for name, got, want in (("dgate", dgu[:, :ff], gf.grad), ("dup", dgu[:, ff:], uf.grad)):
        assert not torch.isnan(got.float()).any(), name
        err = (got.double() - want).abs().max().item()
        assert err < 2e-2 * max(1.0, want.abs().max().item()), f"{name}: {err}"


# ------------------------------------------------------------------------------------------------ model
CFG = dict(H.MT5_SMALL, num_layers=2, num_decoder_layers=3)


def _hf(p, cfg=CFG, seed=0):
    from transformers import MT5Config, MT5ForConditionalGeneration as HFMT5
    torch.manual_seed(seed)
    config = MT5Config(dropout_rate=p, feed_forward_proj="gated-gelu", attn_implementation="eager", decoder_start_token_id=0,
                       pad_token_id=0, **cfg)
    return H._bf16_exact_(HFMT5(config).train())


def _mine(ref, config=None):
    m = MT5ForConditionalGeneration(config or ref.config, device=DEV)
    m.load_reference_state_dict(ref.state_dict())
    return m


def _cuda(b):
    return {k: v.cuda() for k, v in b.items()}


def _grad_close(got, want, name):
    cos = torch.dot(got.flatten(), want.flatten()) / (got.norm() * want.norm() + 1e-30)
    assert cos.item() >= 0.998, (name, cos.item())
    assert abs(got.norm().item() / (want.norm().item() + 1e-30) - 1.0) <= 0.03, (name, got.norm().item(), want.norm().item())


@pytest.mark.parametrize("tied", [True, False])
def test_model_parity_with_replayed_masks(tied, monkeypatch):
    rate = 0.1
    ref = _hf(rate)
    config = ref.config
    sd = dict(ref.state_dict())
    if not tied:
        config = copy.copy(ref.config)
        config.tie_word_embeddings = False
        sd["lm_head.weight"] = ref.shared.weight.detach().clone()
    mine = MT5ForConditionalGeneration(config, device=DEV)
    mine.load_reference_state_dict(sd)
    B, Se, Sd = 2, 96, 40
    batch = H.make_t5_batch(CFG["vocab_size"], B, Se, Sd, seed=7, pad_tail=13)
    sites = site_table(CFG["num_layers"], CFG["num_decoder_layers"], B, Se, Sd, CFG["d_model"], CFG["num_heads"], CFG["d_ff"])
    assert mine.dropout_sites == len(sites)
    seed = mine.dropout_seed
    calls = []

    def replay(x, p=0.5, training=True, inplace=False):
        site, kind, shape = sites[len(calls)]
        assert tuple(x.shape) == shape and p == rate, (site, tuple(x.shape), shape)
        if kind == "hidden":
            keep = R.hidden_keep(seed, site, shape[0] * shape[1], shape[2], p).reshape(shape)
        else:
            keep = R.attn_keep(seed, site, *shape, p)
        calls.append(site)
        return x * torch.from_numpy(keep).to(x.dtype) / (1.0 - p)

    monkeypatch.setattr(torch.nn.functional, "dropout", replay)
    out_ref = ref(**batch)
    assert len(calls) == len(sites)
    out_ref.loss.backward()
    monkeypatch.undo()
    out = mine(**_cuda(batch), return_logits=True)
    assert int(mine.dropout_counter.item()) == mine.dropout_sites
    assert abs(out.loss.item() - out_ref.loss.item()) <= 3e-3 + 5e-4 * abs(out_ref.loss.item()), \
        (out.loss.item(), out_ref.loss.item())
    tol = 4 * 2.0 ** -8 * out_ref.logits.abs().max().item()
    assert (out.logits.float().cpu() - out_ref.logits.detach()).abs().max().item() <= tol
    out.loss.backward()
    torch.cuda.synchronize()
    refp = dict(ref.named_parameters())
    checked = 0
    for name, prm in mine.named_parameters():
        got = prm.main_grad.float().cpu()
        if name == "lm_head.weight":      # untied: the head and the embedding together carry HF's tied gradient
            continue
        if name == "shared.weight" and not tied:
            got = got + mine.P("lm_head.weight").main_grad.float().cpu()
        _grad_close(got, refp[name].grad, name)
        checked += 1
    assert checked == len(refp)
    assert "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight" in refp
    assert "decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight" in refp


def _loss_grads(torch_seed, batch, p=0.1):
    ref = _hf(p)
    torch.manual_seed(torch_seed)       # the dropout seed is drawn at construction
    m = _mine(ref)
    out = m(**_cuda(batch))
    out.loss.backward()
    torch.cuda.synchronize()
    return out.loss.item(), torch.cat([q.main_grad.flatten().float() for q in m._p.values()])


def test_determinism_and_seed_dependence():
    batch = H.make_t5_batch(CFG["vocab_size"], 2, 64, 32, seed=9, pad_tail=5)
    l1, g1 = _loss_grads(17, batch)
    l2, g2 = _loss_grads(17, batch)
    l3, g3 = _loss_grads(18, batch)
    assert l1 == l2 and torch.equal(g1, g2)
    assert l1 != l3 and not torch.equal(g1, g3)


def test_eval_mode_equals_dropout_free_config_and_train_mode_no_grad_drops():
    ref = _hf(0.1)
    cfg0 = copy.copy(ref.config)
    cfg0.dropout_rate = 0.0
    mine, plain = _mine(ref), _mine(ref, cfg0)
    assert plain.dropout_counter is None
    batch = _cuda(H.make_t5_batch(CFG["vocab_size"], 2, 64, 32, seed=4, pad_tail=7))
    mine.eval(); plain.eval()
    a = mine(**batch, return_logits=True)
    b = plain(**batch, return_logits=True)
    assert torch.equal(a.logits, b.logits) and a.loss.item() == b.loss.item()
    a.loss.backward(); b.loss.backward()
    torch.cuda.synchronize()
    grads = lambda m: torch.cat([q.main_grad.flatten() for q in m._p.values()])
    assert torch.equal(grads(mine), grads(plain))
    assert int(mine.dropout_counter.item()) == 0             # eval draws no masks
    mine.train()
    with torch.no_grad():
        c = mine(**batch, return_logits=True)
        assert int(mine.dropout_counter.item()) == mine.dropout_sites
        d = mine(**batch, return_logits=True)                 # the next micro-batch: fresh masks
    assert not torch.equal(c.logits, b.logits) and not torch.equal(c.logits, d.logits)
    assert int(mine.dropout_counter.item()) == 2 * mine.dropout_sites


def _graph_vs_eager(stage, ga, p):
    from fsb200.trainer import PretrainStep
    runs = []
    for graph in (False, True):
        torch.manual_seed(3)
        model = _mine(_hf(p))
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, weight_decay=0.01, grad_clip=1.0, ga_steps=ga, stage=stage,
                          cuda_graph=graph)
        losses = []
        for it in range(5):
            # no attention_mask: the forward reads whether a padding mask is needed on the host, which a capture cannot do
            mbs = [{k: v.cuda() for k, v in H.make_t5_batch(CFG["vocab_size"], 2, 64, 32, seed=50 + 2 * it + m).items()
                    if k != "attention_mask"} for m in range(ga)]
            losses.append(float(st.step_device(mbs)))
        runs.append((losses, model.flat.params.clone(), int(model.dropout_counter.item()), model.dropout_sites))
    return runs


@pytest.mark.parametrize("stage,ga", [(1, 1), (2, 1), (1, 2)])
def test_cuda_graph_step_equals_eager_with_dropout(stage, ga):
    (l0, p0, c0, sites), (l1, p1, c1, _) = _graph_vs_eager(stage, ga, 0.1)
    assert c0 == c1 == 5 * ga * sites
    assert max(abs(a - b) for a, b in zip(l0, l1)) < 1e-5, (l0, l1)
    assert torch.equal(p0, p1), (p0.float() - p1.float()).abs().max()


def test_generate_eval_equals_dropout_free_and_training_mode_raises():
    ref = _hf(0.1)
    mine = _mine(ref)
    cfg0 = copy.copy(ref.config)
    cfg0.dropout_rate = 0.0
    plain = _mine(ref, cfg0)
    ids = H.make_t5_batch(CFG["vocab_size"], 2, 40, 8, seed=3)["input_ids"].cuda()
    with pytest.raises(RuntimeError, match="eval"):
        mine.generate(ids, max_length=12)
    mine.eval(); plain.eval()
    a = mine.generate(ids, max_length=12)
    b = plain.generate(ids, max_length=12)
    assert torch.equal(a, b)
    c = mine.generate(ids, max_length=12, num_beams=2)
    d = plain.generate(ids, max_length=12, num_beams=2)
    assert torch.equal(c, d)


def test_dropout_rate_outside_unit_interval_is_rejected():
    ref = _hf(0.0)
    cfg = copy.copy(ref.config)
    for bad in (1.0, -0.1):
        cfg.dropout_rate = bad
        with pytest.raises(RuntimeError, match="outside"):
            MT5ForConditionalGeneration(cfg, device=DEV)


# ------------------------------------------------------------------------------------------------ recipe
@pytest.fixture
def launched(monkeypatch):
    import hf_fixtures as F
    monkeypatch.syspath_prepend(os.path.join(F.ROOT, "fengshen-lm_b200"))
    saved_path = list(sys.path)
    import fsb200.hf as hf
    import fsb200.launch as launch
    import hf_recipes as RC
    launch.prepare(RC.EXAMPLE)
    yield hf
    hf.uninstall()
    sys.path[:] = saved_path


def test_t5_recipe_with_dropout_trains_exports_and_resumes(launched, tmp_path, monkeypatch):
    """The released mT5 / Randeng configs carry dropout_rate 0.1: the pretrain_t5.py structure runs on such a config."""
    import hf_fixtures as F
    import hf_recipes as RC
    monkeypatch.setattr(F, "MT5_CFG", dict(F.MT5_CFG, dropout_rate=0.1))
    trainer, module = RC.t5_recipe(tmp_path, min_drop=5.0)
    assert type(module.model).__module__ == "fsb200.hf" and module.model.flat.params.is_cuda
    assert module.model.p_drop == 0.1 and int(module.model.dropout_counter.item()) > 0
