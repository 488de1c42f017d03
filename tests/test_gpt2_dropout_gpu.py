"""GPU: GPT-2 dropout — the model against transformers' GPT2LMHeadModel on replayed masks, in CUDA graphs, in generation, in
the Wenzhong recipe and in a per-launch fp64 census at C2 width (its causal attention against fp64:
tests/test_attention_dropout_gpu.py). Every mask is rebuilt by the numpy Philox of tests/philox_ref.py from the layout
documented in include/fsb200.h, never read from the library."""
import copy
import gc
import math
import os
import sys
import time

import pytest
import torch

import philox_ref as R
from test_gpt2_dropout_cpu import site_table

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)

from fsb200 import ops  # noqa: E402
from fsb200.models.gpt2 import GPT2LMHeadModel  # noqa: E402

DEV = "cuda"


# ------------------------------------------------------------------------------------------------ model
CFG = dict(H.GPT2_SMALL, n_layer=3)


def _hf(pe, pa, pr, cfg=CFG, seed=0):
    from transformers import GPT2Config, GPT2LMHeadModel as HFGPT2
    torch.manual_seed(seed)
    config = GPT2Config(embd_pdrop=pe, attn_pdrop=pa, resid_pdrop=pr, activation_function="gelu_new",
                        attn_implementation="eager", bos_token_id=3, eos_token_id=3, **cfg)
    return H._bf16_exact_(HFGPT2(config).train())


def _mine(ref, config=None):
    m = GPT2LMHeadModel(config or ref.config, device=DEV)
    m.load_reference_state_dict(ref.state_dict())
    return m


def _cfg0(ref):
    c = copy.copy(ref.config)
    c.embd_pdrop = c.attn_pdrop = c.resid_pdrop = 0.0
    return c


def _batch(B, S, seed, pad=(0, 13)):
    """A causal-LM batch whose rows are right-padded by `pad` tokens (labels -100 there)."""
    b = H.make_lm_batch(CFG["vocab_size"], B, S, seed=seed)
    for r, n in enumerate(pad):
        if n:
            b["attention_mask"][r, S - n:] = 0
            b["labels"][r, S - n:] = -100
    return b


def _cuda(b):
    return {k: v.cuda() for k, v in b.items()}


def _grads(m):
    return torch.cat([q.main_grad.flatten().float() for q in m._p.values()])


@pytest.mark.parametrize("probs", [(0.1, 0.2, 0.05), (0.1, 0.0, 0.1)], ids=["distinct", "attn0"])
def test_model_parity_with_replayed_masks(probs, monkeypatch):
    ref = _hf(*probs)
    mine = _mine(ref)
    B, S = 3, 96
    batch = _batch(B, S, seed=5, pad=(0, 13, 40))
    sites = site_table(CFG["n_layer"], B, S, CFG["n_embd"], CFG["n_head"], *probs)
    assert mine.dropout_sites == len(sites)
    seed = mine.dropout_seed
    calls = []

    def replay(x, p=0.5, training=True, inplace=False):
        site, kind, shape, wp = sites[len(calls)]
        assert tuple(x.shape) == shape and p == wp, (site, tuple(x.shape), shape, p, wp)
        calls.append(site)
        if p == 0.0:
            return x
        if kind == "hidden":
            keep = R.hidden_keep(seed, site, shape[0] * shape[1], shape[2], p).reshape(shape)
        else:
            keep = R.attn_keep(seed, site, *shape, p)
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
    for name, prm in mine.named_parameters():      # transformer.wte.weight carries the tied LM head's gradient too
        got, want = prm.main_grad.float().cpu(), refp[name].grad
        cos = torch.dot(got.flatten(), want.flatten()) / (got.norm() * want.norm() + 1e-30)
        assert cos.item() >= 0.998, (name, cos.item())
        assert abs(got.norm().item() / (want.norm().item() + 1e-30) - 1.0) <= 0.03, (name, got.norm().item(), want.norm().item())
        checked += 1
    assert checked == len(refp)


def _loss_grads(torch_seed, batch):
    ref = _hf(0.1, 0.1, 0.1)
    torch.manual_seed(torch_seed)       # the dropout seed is drawn at construction
    m = _mine(ref)
    out = m(**_cuda(batch))
    out.loss.backward()
    torch.cuda.synchronize()
    return out.loss.item(), _grads(m)


def test_determinism_and_seed_dependence():
    batch = _batch(2, 64, seed=9)
    l1, g1 = _loss_grads(17, batch)
    l2, g2 = _loss_grads(17, batch)
    l3, g3 = _loss_grads(18, batch)
    assert l1 == l2 and torch.equal(g1, g2)
    assert l1 != l3 and not torch.equal(g1, g3)


def test_eval_mode_equals_dropout_free_config_and_train_mode_no_grad_drops():
    ref = _hf(0.1, 0.1, 0.1)
    mine, plain = _mine(ref), _mine(ref, _cfg0(ref))
    assert plain.dropout_counter is None
    batch = _cuda(_batch(2, 64, seed=4, pad=(0, 7)))
    mine.eval(); plain.eval()
    a = mine(**batch, return_logits=True)
    b = plain(**batch, return_logits=True)
    assert torch.equal(a.logits, b.logits) and a.loss.item() == b.loss.item()
    a.loss.backward(); b.loss.backward()
    torch.cuda.synchronize()
    assert torch.equal(_grads(mine), _grads(plain))
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
        model = _mine(_hf(p, p, p))
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, weight_decay=0.01, grad_clip=1.0, ga_steps=ga, stage=stage,
                          cuda_graph=graph)
        losses = []
        for it in range(5):
            # no attention_mask: the forward reads whether a padding mask is needed on the host, which a capture cannot do
            mbs = [{k: v.cuda() for k, v in H.make_lm_batch(CFG["vocab_size"], 2, 64, seed=50 + 2 * it + m).items()
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
    ref = _hf(0.1, 0.1, 0.1)
    mine, plain = _mine(ref), _mine(ref, _cfg0(ref))
    ids = H.make_lm_batch(CFG["vocab_size"], 2, 40, seed=3)["input_ids"].clamp_min(4).cuda()
    with pytest.raises(RuntimeError, match="eval"):
        mine.generate(ids, max_new_tokens=8)
    assert int(mine.dropout_counter.item()) == 0
    mine.eval(); plain.eval()
    assert torch.equal(mine.generate(ids, max_new_tokens=8), plain.generate(ids, max_new_tokens=8))
    assert torch.equal(mine.generate(ids, max_new_tokens=8, num_beams=2), plain.generate(ids, max_new_tokens=8, num_beams=2))
    assert int(mine.dropout_counter.item()) == 0


def test_dropout_probability_outside_unit_interval_is_rejected():
    ref = _hf(0.0, 0.0, 0.0)
    for k in ("embd_pdrop", "attn_pdrop", "resid_pdrop"):
        for bad in (1.0, -0.1):
            cfg = copy.copy(ref.config)
            setattr(cfg, k, bad)
            with pytest.raises(RuntimeError, match="outside"):
                GPT2LMHeadModel(cfg, device=DEV)


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


def test_wenzhong_recipe_with_dropout_trains(launched, tmp_path, monkeypatch):
    """Released GPT-2 / Wenzhong configs carry 0.1 for all three probabilities: finetune_wenzhong.py's structure runs on such
    a config, and its padded batches reach the causal + padding + dropout attention."""
    import hf_fixtures as F
    import hf_recipes as RC
    from pytorch_lightning import Trainer
    monkeypatch.setattr(F, "GPT2_CFG", dict(F.GPT2_CFG, resid_pdrop=0.1, embd_pdrop=0.1, attn_pdrop=0.1))

    def short_qa_files(data_dir, n=48):
        """F.qa_files' format with rows of 10 to 25 bytes, so that every batch of the recipe's max_seq_length 64 is padded"""
        os.makedirs(data_dir, exist_ok=True)
        rows = [{"Question": f"q{i % 7}?" + "x" * (i % 5), "answer": f" rest {i % 3}." + "z" * (i % 11)} for i in range(n)]
        for name in ("train.txt", "valid.txt", "test.txt"):
            with open(os.path.join(data_dir, name), "w", encoding="utf8") as f:
                f.writelines(repr(r) + "\n" for r in rows)
        return rows
    monkeypatch.setattr(F, "qa_files", short_qa_files)
    seen = []
    real_sdpa = ops.sdpa_fwd

    def sdpa(q, k, v, scale, causal, kv_mask=None, drop=None, **kw):
        if causal and drop is not None:
            seen.append((kv_mask is not None, drop.p))
        return real_sdpa(q, k, v, scale, causal, kv_mask=kv_mask, drop=drop, **kw)
    monkeypatch.setattr(ops, "sdpa_fwd", sdpa)
    # the recipe ends by comparing two no_grad forwards of one batch (its padding check); in training mode each would draw
    # its own masks, as transformers' would, so the model is evaluated in eval mode after fit
    real_fit = Trainer.fit

    def fit_then_eval(self, model, *a, **kw):
        out = real_fit(self, model, *a, **kw)
        model.eval()
        return out
    monkeypatch.setattr(Trainer, "fit", fit_then_eval)
    trainer, module = RC.wenzhong_recipe(tmp_path, min_drop=0.5, device="cuda")
    m = module.model
    assert type(m).__module__ == "fsb200.hf" and m.flat.params.is_cuda
    assert (m.p_embd, m.p_attn, m.p_resid) == (0.1, 0.1, 0.1)
    assert int(m.dropout_counter.item()) >= 24 * m.dropout_sites      # every training step drew its masks
    assert (True, 0.1) in seen, seen[:8]


# ------------------------------------------------------------------------------------------------ per-launch census
def test_every_launch_of_a_gpt2_dropout_step_against_fp64(monkeypatch):
    """One GPT-2 training step at C2 width (hidden 768, 12 heads, S 1024, 2 layers) with all three probabilities 0.1 and
    right-padded rows, every launch checked against fp64 (tests/launch_refs.py) as test_path_launches_gpu.py does for the
    BERT / T5 dropout steps; the stream counter is preset to 2^32 - 5 so that base + site carries into the high word."""
    import launch_refs as LR
    from launch_census import DropoutLog, Recorder, dropout_stream_problems, free_gib, site_of
    from test_path_launches_gpu import COUNTER_PRESET, _finish, _run
    import bench
    from fsb200.trainer import PretrainStep
    case = "dropout-gpt2-110m"
    gc.collect(); torch.cuda.empty_cache()
    if free_gib() < 12:
        pytest.skip(f"{case} and its fp64 checks need about 12 GiB free; {free_gib():.1f} GiB are")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    torch.manual_seed(0)
    w = bench.workload("gpt2-110m")
    from types import SimpleNamespace
    cfg = SimpleNamespace(vocab_size=w["vocab_size"], n_positions=w["n_positions"], n_embd=w["n_embd"], n_layer=2,
                          n_head=w["n_head"], layer_norm_epsilon=1e-5, initializer_range=0.02, resid_pdrop=0.1,
                          embd_pdrop=0.1, attn_pdrop=0.1, activation_function="gelu_new")
    dev = torch.device("cuda", torch.cuda.current_device())
    model = GPT2LMHeadModel(cfg, device=dev, world_size=1)
    model.dropout_counter.fill_(COUNTER_PRESET)
    stepper = PretrainStep(model, lambda s_: w["lr"], lr=w["lr"], betas=w["betas"], weight_decay=w["wd"],
                           grad_clip=w["clip"], ga_steps=1, stage=2, cuda_graph=False)
    b = {k: v.to(dev) for k, v in bench.make_host_batches(w, 1, 0)[0].items()}
    am = torch.ones_like(b["input_ids"])
    am[1::2, w["seq"] - 300:] = 0            # every other row right-padded
    b["attention_mask"] = am
    b["labels"] = b["labels"].masked_fill(am == 0, -100)
    log = DropoutLog()
    rec = Recorder(LR.CHECKERS, extra_key=site_of, observe=log.observe)
    loss, growth = _run(monkeypatch, rec, lambda: stepper.step_device([b]))
    _finish(case, rec, growth, t0)
    assert math.isfinite(float(loss.item())), f"{case}: loss {loss.item()}"
    n = model.dropout_sites
    assert log.advances == [(COUNTER_PRESET, n)], f"{case}: dropout_advance calls {log.advances}"
    assert any(b_ + s >= 2 ** 32 for _, b_, s, *_ in log.uses) and any(b_ + s < 2 ** 32 for _, b_, s, *_ in log.uses)
    problems = dropout_stream_problems(log.advances, log.uses)
    assert not problems, f"{case}: " + "; ".join(problems[:5])
    checked_sites = {k[1][-1][1] for k in rec.checked if k[1] and k[1][-1][0] == "extra" and k[1][-1][1] is not None}
    assert checked_sites == set(range(n)), f"{case}: value-checked sites {sorted(checked_sites)}, want range({n})"
    for op in ("sdpa_fwd", "sdpa_bwd"):
        assert any(k[0] == op and ("causal", True) in k[1] and ("drop", "Dropout") in k[1] for k in rec.checked), \
            f"{case}: no causal {op} call carrying a drop was checked"
    del model, stepper, loss
    gc.collect(); torch.cuda.empty_cache()
