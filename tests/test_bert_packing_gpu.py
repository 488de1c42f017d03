"""GPU: BERT / MegatronBERT MLM (+ sentence order) pretraining on packed batches (fsb200/packing.py pack_mlm_batch +
forward(segment_ids=..., cls_positions=...)), with and without dropout.

Parity: every packed sample run alone in transformers (fp32, CPU), at dropout 0.1 with F.dropout replayed from that sample's
sub-blocks of the packed row's masks (rebuilt by tests/philox_ref.py), the loss the MLM mean over every labelled token plus
the sentence-order mean over the samples, at the thresholds of test_dropout_gpu.py. At dropout 0 the packed batch is the
padded batch it came from. Exact: all-zero segment_ids with one [CLS] per row is the unsegmented path; no-grad equals grad;
the CUDA-graph step equals eager on a fixed packed shape. Also the per-launch fp64 and write-footprint censuses of a packed
MegatronBERT dropout step, and examples/pretrain_erlangshen_bert.py --pack_sequences through Trainer.fit, checkpoint and
resume."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

import philox_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hf_oracle as H  # noqa: E402  (checker only)

from fsb200.engine import ZeroEngine  # noqa: E402
from fsb200.models.bert import BertForMaskedLM, MegatronBertForPreTraining  # noqa: E402
from fsb200.packing import pack_mlm_batch  # noqa: E402

pytestmark = pytest.mark.gpu

S = H.BERT_SMALL["max_position_embeddings"]    # 128: the packed row length
V = H.BERT_SMALL["vocab_size"]
PAD, CLS = 0, 1


def _build_pair(cls_name, p, seed=0):
    from transformers import BertConfig, MegatronBertConfig
    import transformers
    cfgcls = BertConfig if cls_name == "bert" else MegatronBertConfig
    torch.manual_seed(seed)
    config = cfgcls(hidden_dropout_prob=p, attention_probs_dropout_prob=p, hidden_act="gelu", attn_implementation="eager",
                    **H.BERT_SMALL)
    ref = (transformers.BertForMaskedLM if cls_name == "bert" else transformers.MegatronBertForPreTraining)(config)
    ref.train()
    H._bf16_exact_(ref)
    mine = (BertForMaskedLM if cls_name == "bert" else MegatronBertForPreTraining)(config, device="cuda")
    mine.load_reference_state_dict(ref.state_dict())
    return ref, mine


def _docs(lengths, seed):
    """An ErLangShenCollator-format batch: one document per row, [CLS] first, token types 0 then 1, labels on ~15 % of the
    non-[CLS] tokens, padded to S with PAD (token type PAD too, labels -100, attention_mask 0), next_sentence_label."""
    rs = np.random.RandomState(seed)
    n = len(lengths)
    ids = torch.full((n, S), PAD, dtype=torch.int64)
    tt = torch.full((n, S), PAD, dtype=torch.int64)
    lab = torch.full((n, S), -100, dtype=torch.int64)
    am = torch.zeros((n, S), dtype=torch.int64)
    for i, m in enumerate(lengths):
        t = torch.from_numpy(rs.randint(2, V, size=m).astype(np.int64))
        t[0] = CLS
        ids[i, :m], am[i, :m] = t, 1
        tt[i, m // 2:m] = 1
        tt[i, :m // 2] = 0
        sel = torch.from_numpy(rs.rand(m) < 0.15)
        sel[0] = False
        lab[i, :m] = torch.where(sel, t, torch.full_like(t, -100))
    nsl = torch.from_numpy(rs.randint(0, 2, size=n).astype(np.int64))
    return {"input_ids": ids, "attention_mask": am, "token_type_ids": tt, "labels": lab, "next_sentence_label": nsl}


def _lengths(n, seed, lo=6, hi=S // 2):
    rs = np.random.RandomState(seed)
    return [int(x) for x in rs.randint(lo, hi, size=n)]


def _cuda(b):
    return {k: v.cuda() for k, v in b.items()}


def _grads(m):
    return {n: q.main_grad.float().cpu().flatten().clone() for n, q in m.named_parameters()}


def _cos(a, b):
    return (torch.dot(a, b) / (a.norm() * b.norm() + 1e-30)).item()


def _run(model, batch, **kw):
    model.flat.grads.zero_()
    out = model(**_cuda(batch), **kw)
    out.loss.backward()
    torch.cuda.synchronize()
    return out, _grads(model)


def _for_model(cls_name, b):
    return b if cls_name == "megatron" else {k: v for k, v in b.items() if k not in ("next_sentence_label", "cls_positions")}


def _samples(padded, packed):
    """(row, start, length) of every sample i of the padded batch inside the packed one, in sample order."""
    n = padded["attention_mask"].sum(1).tolist()
    return [(int(c) // S, int(c) % S, m) for c, m in zip(packed["cls_positions"], n)]


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("cls_name", ["bert", "megatron"])
def test_packed_parity_with_transformers_per_sample(cls_name, p, monkeypatch):
    """Each packed sample against transformers run on that sample alone; at p 0.1 with the packed row's masks replayed."""
    ref, mine = _build_pair(cls_name, p)
    padded = _docs(_lengths(7, seed=1), seed=2)
    packed = pack_mlm_batch(padded, S, PAD)
    B = packed["input_ids"].shape[0]
    assert B < 7
    h, nh, nl = H.BERT_SMALL["hidden_size"], H.BERT_SMALL["num_attention_heads"], H.BERT_SMALL["num_hidden_layers"]
    sites = [("hidden", 0)]
    for i in range(nl):
        sites += [("attn", 1 + 3 * i), ("hidden", 2 + 3 * i), ("hidden", 3 + 3 * i)]
    full = {}
    if p > 0:
        seed = mine.dropout_seed
        full = {site: (R.hidden_keep(seed, site, B * S, h, p).reshape(B, S, h) if kind == "hidden"
                       else R.attn_keep(seed, site, B, nh, S, S, p)) for kind, site in sites}
    nsp = cls_name == "megatron"
    mlm_sum, n_lab, nsp_sum, logits_ref, nsp_ref = 0.0, 0, 0.0, [], []
    ce = torch.nn.functional.cross_entropy
    for i, (r, s, m) in enumerate(_samples(padded, packed)):
        calls = []

        def replay(x, p=0.5, training=True, inplace=False):
            kind, site = sites[len(calls)]
            calls.append(site)
            keep = full[site][r:r + 1, s:s + m] if kind == "hidden" else full[site][r:r + 1, :, s:s + m, s:s + m]
            assert tuple(keep.shape) == tuple(x.shape), (site, keep.shape, x.shape)
            return x * torch.from_numpy(np.ascontiguousarray(keep)).to(x.dtype) / (1.0 - p)
        if p > 0:
            monkeypatch.setattr(torch.nn.functional, "dropout", replay)
        out = ref(input_ids=packed["input_ids"][r:r + 1, s:s + m], token_type_ids=packed["token_type_ids"][r:r + 1, s:s + m])
        monkeypatch.undo()
        assert p == 0 or len(calls) == len(sites)
        lg = out.logits if not nsp else out.prediction_logits
        lab = packed["labels"][r, s:s + m]
        mlm_sum = mlm_sum + ce(lg[0], lab, ignore_index=-100, reduction="sum")
        n_lab += int((lab != -100).sum())
        logits_ref.append(lg.detach()[0])
        if nsp:
            nsp_sum = nsp_sum + ce(out.seq_relationship_logits, packed["next_sentence_label"][i:i + 1], reduction="sum")
            nsp_ref.append(out.seq_relationship_logits.detach()[0])
    loss_ref = mlm_sum / n_lab + (nsp_sum / len(logits_ref) if nsp else 0.0)
    loss_ref.backward()
    out, g = _run(mine, _for_model(cls_name, packed), return_logits=True)
    if p > 0:
        assert int(mine.dropout_counter.item()) == mine.dropout_sites
    assert abs(out.loss.item() - loss_ref.item()) <= 4e-3, (out.loss.item(), loss_ref.item())
    lg = out.logits.float().cpu()
    for (r, s, m), want in zip(_samples(padded, packed), logits_ref):
        assert (lg[r, s:s + m] - want).abs().max().item() <= 4 * 2.0 ** -8 * want.abs().max().item(), (r, s, m)
    if nsp:
        got = out.seq_relationship_logits.float().cpu()
        want = torch.stack(nsp_ref)
        assert (got - want).abs().max().item() <= 4 * 2.0 ** -8 * max(want.abs().max().item(), 1.0)
    refp = dict(ref.named_parameters())
    for name, got in g.items():
        want = refp[name].grad
        if want is None or want.norm().item() < 1e-7:
            assert got.norm().item() < 1e-4, name
            continue
        want = want.flatten()
        assert _cos(got, want) >= 0.998, name
        assert abs(got.norm().item() / (want.norm().item() + 1e-30) - 1.0) <= 0.03, name


@pytest.mark.parametrize("cls_name", ["bert", "megatron"])
def test_dropout_zero_packed_matches_padded(cls_name):
    _, mine = _build_pair(cls_name, 0.0)
    padded = _docs(_lengths(8, seed=3), seed=4)
    packed = pack_mlm_batch(padded, S, PAD)
    o_p, g_p = _run(mine, _for_model(cls_name, packed), return_logits=True)
    o_d, g_d = _run(mine, _for_model(cls_name, padded), return_logits=True)
    assert abs(o_p.loss.item() - o_d.loss.item()) <= 3e-3, (o_p.loss.item(), o_d.loss.item())
    for name in g_p:
        if g_d[name].norm().item() < 1e-7:
            continue
        assert _cos(g_p[name], g_d[name]) >= 0.999, name
    lg_p, lg_d = o_p.logits.float(), o_d.logits.float()
    for i, (r, s, m) in enumerate(_samples(padded, packed)):
        want = lg_d[i, :m]
        assert (lg_p[r, s:s + m] - want).abs().max().item() <= 4 * 2.0 ** -8 * want.abs().max().item(), (i, r, s)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("cls_name", ["bert", "megatron"])
def test_one_segment_per_row_is_the_unsegmented_path_bit_for_bit(cls_name, p):
    batch = _docs([S, S], seed=5)
    runs = []
    for packed in (False, True):
        torch.manual_seed(11)           # the dropout seed is drawn at construction
        _, m = _build_pair(cls_name, p, seed=1)
        kw = {} if not packed else {"segment_ids": torch.zeros((2, S), dtype=torch.int64),
                                    "cls_positions": torch.arange(2) * S}
        out, g = _run(m, _for_model(cls_name, dict(batch, **kw)), return_logits=True)
        runs.append((out.loss.item(), out.logits.clone(), out.seq_relationship_logits, g))
    (l0, lg0, n0, g0), (l1, lg1, n1, g1) = runs
    assert l0 == l1
    assert torch.equal(lg0, lg1)
    assert (n0 is None and n1 is None) or torch.equal(n0, n1)
    assert all(torch.equal(g0[n], g1[n]) for n in g0)


def test_packed_loss_curve_follows_the_padded_curve():
    curves = []
    for pack in (False, True):
        _, model = _build_pair("megatron", 0.0)
        eng = ZeroEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1)
        curve = []
        for it in range(20):
            padded = _docs(_lengths(6, seed=100 + it % 4), seed=200 + it % 4)
            out = model(**_cuda(pack_mlm_batch(padded, S, PAD) if pack else padded))
            out.loss.backward()
            eng.backward_done()
            eng.step(lr=1e-3)
            curve.append(out.loss.item())
        curves.append(curve)
    err = np.abs(np.array(curves[0]) - np.array(curves[1])).max()
    assert err <= 1e-2, (err, curves)
    assert curves[1][-1] < curves[1][0]


def test_no_grad_loss_equals_grad_loss_with_dropout():
    """The same masks (the stream counter rewound): the no-grad forward is the training forward without saving."""
    _, model = _build_pair("megatron", 0.1)
    batch = _cuda(pack_mlm_batch(_docs(_lengths(6, seed=6), seed=7), S, PAD))
    with torch.no_grad():
        l0 = model(**batch).loss.item()
    model.dropout_counter.zero_()
    out = model(**batch)
    assert out.loss.item() == l0
    out.loss.backward()


# every micro-batch packs into exactly two full rows of four documents: a fixed shape for the CUDA graph
_FIXED = [40, 30, 50, 8, 60, 20, 40, 8]


def _fixed_packed(seed):
    p = pack_mlm_batch(_docs(_FIXED, seed=seed), S, PAD)
    assert p["input_ids"].shape == (2, S) and p["cls_positions"].tolist() == [0, 40, 70, 120, 128, 188, 208, 248]
    return _cuda(p)


def _graph_vs_eager(stage, ga):
    from fsb200.trainer import PretrainStep
    runs = []
    for graph in (False, True):
        torch.manual_seed(3)
        _, model = _build_pair("megatron", 0.1)
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, weight_decay=0.01, grad_clip=1.0, ga_steps=ga, stage=stage,
                          cuda_graph=graph)
        losses = []
        for it in range(4):
            losses.append(float(st.step_device([_fixed_packed(300 + ga * it + m) for m in range(ga)])))
        runs.append((losses, model.flat.params.clone(), int(model.dropout_counter.item()), model.dropout_sites))
    return runs


@pytest.mark.parametrize("stage,ga", [(1, 2), (2, 1)])
def test_cuda_graph_step_equals_eager_on_packed_batches_with_dropout(stage, ga):
    (l0, p0, c0, sites), (l1, p1, c1, _) = _graph_vs_eager(stage, ga)
    assert c0 == c1 == 4 * ga * sites
    assert l0 == l1, (l0, l1)
    assert torch.equal(p0, p1)


def test_cuda_graph_zero2_ga2_on_packed_batches_reported():
    """ZeRO-2 with GA 2: reported, not asserted (the unpacked BERT step's graph-vs-eager difference there is a recorded
    expected failure)."""
    (l0, p0, _, _), (l1, p1, _, _) = _graph_vs_eager(2, 2)
    diff = (p0.float() - p1.float()).abs().max().item()
    print(f"packed MegatronBERT ZeRO-2 GA 2 graph vs eager: losses equal {l0 == l1}, params equal {torch.equal(p0, p1)}, "
          f"max |param difference| {diff:.3g}")
    assert all(math.isfinite(x) for x in l0 + l1)


def test_refusals():
    _, model = _build_pair("megatron", 0.1)
    packed = pack_mlm_batch(_docs(_lengths(6, seed=8), seed=9), S, PAD)
    bad = packed["attention_mask"].clone()
    bad[0, -1] = 0
    with pytest.raises(ValueError, match="attention_mask has zeros"):
        model(**dict(_cuda(packed), attention_mask=bad))          # a host mask: checked exactly
    with pytest.raises(ValueError, match="need cls_positions"):
        model(**{k: v for k, v in _cuda(packed).items() if k != "cls_positions"})
    with pytest.raises(ValueError, match="segment_ids must be"):
        model(**dict(_cuda(packed), segment_ids=packed["segment_ids"][:, :-1].cuda()))
    out = model(**_cuda(packed))          # an all-ones device mask passes (checked asynchronously)
    assert math.isfinite(out.loss.item())
    # without next_sentence_label and cls_positions: MLM only, no sentence-order logits
    out = model(**{k: v for k, v in _cuda(packed).items() if k not in ("cls_positions", "next_sentence_label")})
    assert out.seq_relationship_logits is None and math.isfinite(out.loss.item())
    from transformers import MegatronBertConfig
    cfg = MegatronBertConfig(**dict(H.BERT_SMALL, num_attention_heads=2))      # head_dim 128
    m128 = MegatronBertForPreTraining(cfg, device="cuda")
    with pytest.raises(ValueError, match="head_dim 64"):
        m128(**_cuda(packed))


# ---------------------------------------------------------------------------------------- per-launch censuses
def _ref_attention(q, k, v, scale, seg_start, seg_end, b, causal, drop_mult):
    qf, kf, vf = (t[b].double().permute(1, 0, 2).detach().requires_grad_(True) for t in (q, k, v))
    kk = torch.arange(q.shape[1], device=q.device)
    vis = (kk[None, :] >= seg_start[b].long()[:, None]) & (kk[None, :] < seg_end[b].long()[:, None])
    if causal:
        vis &= kk[None, :] <= kk[:, None]
    s = (scale * qf @ kf.transpose(-1, -2)).masked_fill(~vis, float("-inf"))
    return (torch.softmax(s, -1) * drop_mult) @ vf, s, (qf, kf, vf)


def check_sdpa_segments_fwd(real, bound, q, k, v, scale, seg_start, seg_end, out=None, drop=None, causal=True):
    """Every row whole against fp64 under its block-diagonal (causal or bidirectional) pattern and the keep mask at the
    row-relative (q, k)."""
    import launch_refs as LR
    o, lse = ret = real(q, k, v, scale, seg_start, seg_end, out=out, drop=drop, causal=causal)
    d = None if drop is None else LR.drop_spec(drop)
    for b in range(q.shape[0]):
        m = 1.0 if d is None else LR.attn_mult(d, range(b, b + 1), q.shape[2], q.shape[1], k.shape[1], q.device)[0]
        ref, s, _ = _ref_attention(q, k, v, scale, seg_start, seg_end, b, causal, m)
        bound.close("O", o[b].permute(1, 0, 2), ref.detach(), 2e-2 * max(1.0, ref.abs().max().item() / 4))
        bound.close("lse", lse[b].double() * math.log(2.0), torch.logsumexp(s, -1).detach(), 2e-3)
    return ret


def check_sdpa_segments_bwd(real, bound, q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv, drop=None,
                            causal=True):
    import launch_refs as LR
    ret = real(q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv, drop=drop, causal=causal)
    d = None if drop is None else LR.drop_spec(drop)
    for b in range(q.shape[0]):
        m = 1.0 if d is None else LR.attn_mult(d, range(b, b + 1), q.shape[2], q.shape[1], k.shape[1], q.device)[0]
        with torch.enable_grad():     # the step's backward runs with autograd recording off
            ref, _, (qf, kf, vf) = _ref_attention(q, k, v, scale, seg_start, seg_end, b, causal, m)
            ref.backward(dout[b].double().permute(1, 0, 2))
        for name, got, want in (("dQ", dq, qf.grad), ("dK", dk, kf.grad), ("dV", dv, vf.grad)):
            bound.close(name, got[b].permute(1, 0, 2), want, 3e-2 * max(1.0, want.abs().max().item()))
    return ret


def _packed_dropout_census(monkeypatch, checkers):
    """One packed MegatronBERT training step at dropout 0.1, GA 2, every op launch recorded and its first call of each
    signature checked by `checkers`; returns the recorder."""
    from launch_census import Recorder
    from fsb200 import lib as L
    from fsb200.trainer import PretrainStep
    torch.manual_seed(5)
    _, model = _build_pair("megatron", 0.1)
    st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2)
    mbs = [_cuda(pack_mlm_batch(_docs(_lengths(6, seed=60 + m), seed=70 + m), S, PAD)) for m in range(2)]
    rec = Recorder(checkers)
    rec.install(monkeypatch)
    c0 = L.launch_count
    try:
        loss = st.step_device(mbs)
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    ops_seen = {key[0] for key in rec.calls}
    assert {"segment_bounds", "sdpa_segments_fwd", "sdpa_segments_bwd"} <= ops_seen
    assert "sdpa_fwd" not in ops_seen and "sdpa_bwd" not in ops_seen
    for op in ("sdpa_segments_fwd", "sdpa_segments_bwd"):
        assert any(k[0] == op and ("drop", "Dropout") in k[1] for k in rec.checked), f"no {op} carrying a drop was checked"
    assert L.launch_count - c0 - rec.extra_launches == rec.wrapped_launches
    assert math.isfinite(float(loss.item()))
    return rec


def test_every_launch_of_a_packed_dropout_step_against_fp64(monkeypatch):
    import launch_refs as LR
    import test_llama_packing_gpu as LP
    checkers = dict(LR.CHECKERS)
    checkers.update(segment_bounds=LP.check_segment_bounds, sdpa_segments_fwd=check_sdpa_segments_fwd,
                    sdpa_segments_bwd=check_sdpa_segments_bwd)
    _packed_dropout_census(monkeypatch, checkers)


def test_write_footprint_of_every_launch_of_a_packed_dropout_step(monkeypatch):
    import footprint as F
    stats = F.Stats()
    _packed_dropout_census(monkeypatch, F.footprint_checkers(stats))
    assert {"sdpa_segments_fwd", "sdpa_segments_bwd"} <= set(stats.checked)


# ---------------------------------------------------------------------------------------- the Erlangshen recipe
@pytest.fixture
def launched(monkeypatch):
    import hf_recipes
    monkeypatch.syspath_prepend(os.path.join(ROOT, "fengshen-lm_b200"))
    saved_path = list(sys.path)
    import fsb200.hf as hf
    import fsb200.launch as launch
    launch.prepare(hf_recipes.EXAMPLE)
    yield hf
    hf.uninstall()
    sys.path[:] = saved_path


def test_erlangshen_example_with_pack_sequences_trains_checkpoints_and_resumes(launched, tmp_path, monkeypatch):
    """examples/pretrain_erlangshen_bert.py --pack_sequences under the recipe's ZeRO-1 DeepSpeed JSON, Python and native
    collators: one epoch, then a resumed second; every batch the model saw was packed."""
    import runpy
    import hf_fixtures as F
    import bert_collator_cases as C
    F.bert_dir(tmp_path / "m")
    corpus = tmp_path / "train.json"             # one paragraph per document (11 to 53 tokens): several share a row of 64
    docs = [t for t in C.TEXTS if "。" in t]
    with open(corpus, "w", encoding="utf8") as f:
        for i in range(64):
            f.write(json.dumps({"text": docs[i % len(docs)]}, ensure_ascii=False) + "\n")
    ds_json = tmp_path / "ds_config.json"
    ds_json.write_text(json.dumps({"zero_optimization": {"stage": 1}, "bf16": {"enabled": True}, "gradient_clipping": 2,
                                   "train_micro_batch_size_per_gpu": 8}))
    monkeypatch.setenv("PL_DEEPSPEED_CONFIG_PATH", str(ds_json))
    import hf_recipes
    ns = runpy.run_path(hf_recipes.EXAMPLE, run_name="example_not_main")
    seen = []
    fwd = ns["ErLangShenBert"].forward

    def spy(self, **batch):
        seen.append({k: tuple(v.shape) for k, v in batch.items()})
        return fwd(self, **batch)
    monkeypatch.setattr(ns["ErLangShenBert"], "forward", spy)

    def argv(epochs, native):
        return ["--model_path", str(tmp_path / "m"), "--train_file", str(corpus), "--train_batchsize", "8",
                "--max_seq_length", "64", "--max_epoch", str(epochs), "--learning_rate", "1e-3", "--weight_decay", "0.1",
                "--warmup_ratio", "0.1", "--strategy", "deepspeed_stage_1", "--replace_sampler_ddp", "False",
                "--dataloader_workers", "0", "--log_every_n_steps", "1", "--default_root_dir", str(tmp_path),
                "--save_ckpt_path", str(tmp_path / "ckpt"), "--load_ckpt_path", str(tmp_path / "ckpt" / "last.ckpt"),
                "--save_last", "--every_n_train_steps", "4", "--precision", "bf16", "--pack_sequences"] + \
            (["--native_collator"] if native else [])

    trainer, module = ns["main"](argv(1, False))
    assert type(module.model).__module__ == "fsb200.hf"
    assert trainer.global_step == 8
    assert all({"segment_ids", "position_ids", "cls_positions"} <= set(b) for b in seen)
    assert any(b["input_ids"][0] < 8 for b in seen)                 # documents shared rows
    losses = [json.loads(line)["train_loss"] for line in open(os.path.join(trainer.logger.save_dir, "metrics.jsonl"))]
    assert all(math.isfinite(x) for x in losses)
    ck = tmp_path / "ckpt" / "last.ckpt" / "checkpoint"
    state = torch.load(ck / "mp_rank_00_model_states.pt", map_location="cpu", weights_only=False)
    assert state["global_step"] == 8 and state["global_samples"] == 64
    w_before = module.model.flat.params.clone()
    seen.clear()
    trainer2, module2 = ns["main"](argv(2, True))                   # resumed, on the native collator
    assert trainer2.global_step == 16 and module2.consumed_samples == 64
    assert seen and all("cls_positions" in b for b in seen)
    assert not torch.equal(module2.model.flat.params, w_before)
