"""GPU: GPT-2 / Wenzhong on packed batches (fsb200/packing.py + GPT2LMHeadModel.forward(segment_ids=...)), with dropout.

Parity: every packed sample run alone in transformers' GPT2LMHeadModel (fp32, CPU) with F.dropout replayed from that
sample's sub-blocks of the packed row's masks (rebuilt by tests/philox_ref.py), the loss the target-weighted mean of the
samples' losses, at the thresholds of test_gpt2_dropout_gpu.py. At dropout 0 the packed batch is the padded batch it came
from. Exact: all-zero segment_ids is the unsegmented path; the model ignores segment-start labels by itself; no-grad equals
grad; the CUDA-graph step equals eager under ZeRO-1 / ZeRO-2 with GA 2 at dropout 0.1. Also the per-launch fp64 and write
footprint censuses of a packed dropout step, and finetune_wenzhong.py's structure with PackingCollator through Trainer.fit,
checkpoint and resume."""
import math
import os
import random

import numpy as np
import pytest
import torch

import philox_ref as R
from test_gpt2_dropout_cpu import site_table
from test_gpt2_dropout_gpu import CFG, _hf, _mine, launched  # noqa: F401  (launched: the recipe's fixture)

from fsb200.engine import ZeroEngine
from fsb200.packing import pack_causal_lm_batch

pytestmark = pytest.mark.gpu

EOS = 3             # the test models' eos (_hf: eos_token_id=3), also the pad, as in GPT2QADataset
S = CFG["n_positions"]


def _qa_padded(n, seed, max_len=S // 3):
    """n question + answer samples padded to S with eos, labels -100 on the pads, attention_mask 0 there: the format of
    GPT2QADataset.encode (padding='max_length')."""
    rng = random.Random(seed)
    ids = torch.full((n, S), EOS, dtype=torch.int64)
    labels = torch.full((n, S), -100, dtype=torch.int64)
    mask = torch.zeros((n, S), dtype=torch.int64)
    for i in range(n):
        m = rng.randint(4, max_len)
        t = torch.tensor([rng.randrange(4, CFG["vocab_size"]) for _ in range(m)])
        ids[i, :m], labels[i, :m], mask[i, :m] = t, t, 1
    return {"input_ids": ids, "labels": labels, "attention_mask": mask}


def _samples(packed):
    """(row, start, end) of every sample of a packed batch (its pad tails, without labels, left out)."""
    out = []
    for r, row in enumerate(packed["segment_ids"].tolist()):
        s = 0
        for t in range(1, S + 1):
            if t == S or row[t] != row[t - 1]:
                if (packed["labels"][r, s:t] != -100).any():
                    out.append((r, s, t))
                s = t
    return out


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


def test_packed_parity_with_transformers_on_replayed_masks(monkeypatch):
    probs = (0.1, 0.2, 0.05)
    ref = _hf(*probs)
    mine = _mine(ref)
    packed = pack_causal_lm_batch(_qa_padded(8, seed=1), S, EOS)
    B = packed["input_ids"].shape[0]
    assert B < 8
    nl, h, nh = CFG["n_layer"], CFG["n_embd"], CFG["n_head"]
    sites = site_table(nl, B, S, h, nh, *probs)
    seed = mine.dropout_seed
    full = {site: (R.hidden_keep(seed, site, B * S, h, p).reshape(B, S, h) if kind == "hidden"
                   else R.attn_keep(seed, site, B, nh, S, S, p)) for site, kind, _, p in sites if p > 0}
    samples = _samples(packed)
    total, n_all, logits_ref = 0.0, 0, []
    for r, s, e in samples:
        calls = []

        def replay(x, p=0.5, training=True, inplace=False):
            site, kind, _, wp = sites[len(calls)]
            assert p == wp
            calls.append(site)
            if p == 0.0:
                return x
            keep = full[site][r:r + 1, s:e] if kind == "hidden" else full[site][r:r + 1, :, s:e, s:e]
            assert tuple(keep.shape) == tuple(x.shape), (site, keep.shape, x.shape)
            return x * torch.from_numpy(np.ascontiguousarray(keep)).to(x.dtype) / (1.0 - p)
        monkeypatch.setattr(torch.nn.functional, "dropout", replay)
        lab = packed["labels"][r:r + 1, s:e]
        out = ref(input_ids=packed["input_ids"][r:r + 1, s:e], position_ids=torch.arange(e - s)[None], labels=lab)
        monkeypatch.undo()
        assert len(calls) == len(sites)
        n = int((lab[0, 1:] != -100).sum())
        total, n_all = total + out.loss * n, n_all + n
        logits_ref.append(out.logits.detach()[0])
    loss_ref = total / n_all
    loss_ref.backward()
    out, g = _run(mine, packed, return_logits=True)
    assert int(mine.dropout_counter.item()) == mine.dropout_sites
    assert abs(out.loss.item() - loss_ref.item()) <= 3e-3 + 5e-4 * abs(loss_ref.item()), (out.loss.item(), loss_ref.item())
    lg = out.logits.float().cpu()
    for (r, s, e), want in zip(samples, logits_ref):
        tol = 4 * 2.0 ** -8 * want.abs().max().item()
        assert (lg[r, s:e] - want).abs().max().item() <= tol, (r, s, e)
    refp = dict(ref.named_parameters())
    for name, got in g.items():
        want = refp[name].grad.flatten()
        assert _cos(got, want) >= 0.998, name
        assert abs(got.norm().item() / (want.norm().item() + 1e-30) - 1.0) <= 0.03, name
    assert len(g) == len(refp)


def test_dropout_zero_packed_matches_padded():
    ref = _hf(0.0, 0.0, 0.0)
    mine = _mine(ref)
    padded = _qa_padded(8, seed=2)
    packed = pack_causal_lm_batch(padded, S, EOS)
    o_p, g_p = _run(mine, packed, return_logits=True)
    o_d, g_d = _run(mine, padded, return_logits=True)
    assert abs(o_p.loss.item() - o_d.loss.item()) <= 3e-3, (o_p.loss.item(), o_d.loss.item())
    for name in g_p:
        assert _cos(g_p[name], g_d[name]) >= 0.999, name
    # each sample in the packed rows sits where the padded batch's row i begins: the samples keep their order
    lg_p, lg_d = o_p.logits.float(), o_d.logits.float()
    samples = _samples(packed)
    kept = [i for i in range(8) if (padded["labels"][i] != -100).any()]
    order = {}
    for (r, s, e) in samples:
        i = next(i for i in kept if i not in order.values() and
                 torch.equal(padded["input_ids"][i, :e - s], packed["input_ids"][r, s:e]))
        order[(r, s, e)] = i
        want = lg_d[i, :e - s]
        assert (lg_p[r, s:e] - want).abs().max().item() <= 4 * 2.0 ** -8 * want.abs().max().item(), (r, s, e)
    assert len(order) == len(kept)


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_zero_segment_ids_is_the_unsegmented_path_bit_for_bit(p):
    ref = _hf(p, p, p)
    batch = {k: v for k, v in _qa_padded(2, seed=5, max_len=S).items()}
    batch["attention_mask"] = torch.ones_like(batch["input_ids"])
    runs = []
    for seg in (None, torch.zeros_like(batch["input_ids"])):
        torch.manual_seed(11)           # the dropout seed is drawn at construction
        m = _mine(ref)
        out, g = _run(m, batch, **({} if seg is None else {"segment_ids": seg}))
        runs.append((out.loss.item(), g))
    (l0, g0), (l1, g1) = runs
    assert l0 == l1
    assert all(torch.equal(g0[n], g1[n]) for n in g0)


def test_model_ignores_segment_start_labels_itself():
    torch.manual_seed(12)
    ref = _hf(0.1, 0.1, 0.1)
    packed = pack_causal_lm_batch(_qa_padded(8, seed=21), S, EOS)
    raw = dict(packed, labels=packed["labels"].clone())
    seg = packed["segment_ids"]
    starts = torch.ones_like(seg, dtype=torch.bool)
    starts[:, 1:] = seg[:, 1:] != seg[:, :-1]
    raw["labels"][starts] = packed["input_ids"][starts]       # a (wrong) target on every segment start
    assert (raw["labels"] != packed["labels"]).any()
    runs = []
    for b in (packed, raw):
        torch.manual_seed(13)
        m = _mine(ref)
        out, g = _run(m, b)
        runs.append((out.loss.item(), g))
    assert runs[0][0] == runs[1][0]
    assert all(torch.equal(runs[0][1][n], runs[1][1][n]) for n in runs[0][1])


def test_packed_loss_curve_follows_the_padded_curve():
    ref = _hf(0.0, 0.0, 0.0)
    curves = []
    for pack in (False, True):
        model = _mine(ref)
        eng = ZeroEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1)
        curve = []
        for it in range(20):
            padded = _qa_padded(6, seed=100 + it % 4)
            out = model(**_cuda(pack_causal_lm_batch(padded, S, EOS) if pack else padded))
            out.loss.backward()
            eng.backward_done()
            eng.step(lr=1e-3)
            curve.append(out.loss.item())
        curves.append(curve)
    err = np.abs(np.array(curves[0]) - np.array(curves[1])).max()
    assert err <= 1e-2, (err, curves)


def test_no_grad_loss_equals_grad_loss_with_dropout():
    """The same masks (the stream counter rewound): the no-grad forward is the training forward without saving."""
    model = _mine(_hf(0.1, 0.1, 0.1))
    batch = _cuda(pack_causal_lm_batch(_qa_padded(6, seed=3), S, EOS))
    with torch.no_grad():
        l0 = model(**batch).loss.item()
    model.dropout_counter.zero_()
    out = model(**batch)
    assert out.loss.item() == l0
    out.loss.backward()


@pytest.mark.parametrize("stage", [1, 2])
def test_cuda_graph_step_equals_eager_on_packed_batches_with_dropout(stage):
    """Fixed-shape packed micro-batches [2, S] (segment_ids is one more static batch buffer), GA 2, dropout 0.1."""
    from fsb200.trainer import PretrainStep
    runs = []
    for graph in (False, True):
        torch.manual_seed(3)
        model = _mine(_hf(0.1, 0.1, 0.1))
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2,
                          stage=stage, cuda_graph=graph)
        losses = []
        for it in range(4):
            mbs = []
            for m in range(2):
                p = pack_causal_lm_batch(_qa_padded(12, seed=300 + 2 * it + m), S, EOS)
                mbs.append({k: v[:2].cuda() for k, v in p.items() if k != "attention_mask"})
            losses.append(float(st.step_device(mbs)))
        runs.append((losses, model.flat.params.clone(), int(model.dropout_counter.item())))
    (l0, p0, c0), (l1, p1, c1) = runs
    assert c0 == c1 == 4 * 2 * model.dropout_sites
    assert l0 == l1, (l0, l1)
    assert torch.equal(p0, p1)


def test_refusals():
    model = _mine(_hf(0.1, 0.1, 0.1))
    packed = pack_causal_lm_batch(_qa_padded(6, seed=4), S, EOS)
    bad = packed["attention_mask"].clone()
    bad[0, -1] = 0
    with pytest.raises(ValueError, match="attention_mask has zeros"):
        model(**dict(_cuda(packed), attention_mask=bad))          # a host mask: checked exactly
    with pytest.raises(ValueError, match="segment_ids must be"):
        model(**dict(_cuda(packed), segment_ids=packed["segment_ids"][:, :-1].cuda()))
    # an all-ones mask on the device passes (checked asynchronously, so a CUDA-graph step stays capturable)
    out = model(**_cuda(packed))
    assert math.isfinite(out.loss.item())


# ---------------------------------------------------------------------------------------- per-launch censuses
def _visible(seg_start, b, Sq):
    """bool [Sq, Sq] of row b: key k visible to query q (seg_start[q] <= k <= q)."""
    k = torch.arange(Sq, device=seg_start.device)
    st = seg_start[b].long()
    return (k[None, :] >= st[:, None]) & (k[None, :] <= k[:, None])


def _ref_attention(q, k, v, scale, seg_start, b, drop_mult):
    """fp64 O of row b and the autograd leaves: [H, S, D]."""
    qf, kf, vf = (t[b].double().permute(1, 0, 2).detach().requires_grad_(True) for t in (q, k, v))
    s = (scale * qf @ kf.transpose(-1, -2)).masked_fill(~_visible(seg_start, b, q.shape[1]), float("-inf"))
    p = torch.softmax(s, -1)
    return (p * drop_mult) @ vf, s, (qf, kf, vf)


def check_sdpa_segments_fwd(real, bound, q, k, v, scale, seg_start, seg_end, out=None, drop=None):
    """drop=None: test_llama_packing_gpu's per-segment causal bounds. With a drop, the keep mask is at the row-relative (q, k),
    so each row is checked whole against an fp64 reference under its block-diagonal causal pattern."""
    import launch_refs as LR
    import test_llama_packing_gpu as LP
    if drop is None:
        return LP.check_sdpa_segments_fwd(real, bound, q, k, v, scale, seg_start, seg_end, out=out)
    o, lse = ret = real(q, k, v, scale, seg_start, seg_end, out=out, drop=drop)
    d = LR.drop_spec(drop)
    H = q.shape[2]
    for b in range(q.shape[0]):
        m = LR.attn_mult(d, range(b, b + 1), H, q.shape[1], k.shape[1], q.device)[0]
        ref, s, _ = _ref_attention(q, k, v, scale, seg_start, b, m)
        bound.close("O", o[b].permute(1, 0, 2), ref.detach(),
                    2e-2 * max(1.0, ref.abs().max().item() / 4))
        bound.close("lse", lse[b].double() * math.log(2.0), torch.logsumexp(s, -1).detach(), 2e-3)
    return ret


def check_sdpa_segments_bwd(real, bound, q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv, drop=None):
    import launch_refs as LR
    import test_llama_packing_gpu as LP
    if drop is None:
        return LP.check_sdpa_segments_bwd(real, bound, q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv)
    ret = real(q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv, drop=drop)
    d = LR.drop_spec(drop)
    H = q.shape[2]
    for b in range(q.shape[0]):
        m = LR.attn_mult(d, range(b, b + 1), H, q.shape[1], k.shape[1], q.device)[0]
        with torch.enable_grad():     # the step's backward runs with autograd recording off
            ref, _, (qf, kf, vf) = _ref_attention(q, k, v, scale, seg_start, b, m)
            ref.backward(dout[b].double().permute(1, 0, 2))
        for name, got, want in (("dQ", dq, qf.grad), ("dK", dk, kf.grad), ("dV", dv, vf.grad)):
            bound.close(name, got[b].permute(1, 0, 2), want, 3e-2 * max(1.0, want.abs().max().item()))
    return ret


def _packed_dropout_census(monkeypatch, checkers):
    """One packed GPT-2 training step at dropout 0.1, GA 2, every op launch recorded and its first call of each signature
    checked by `checkers`; returns the recorder."""
    from launch_census import Recorder
    from fsb200 import lib as L
    from fsb200.trainer import PretrainStep
    torch.manual_seed(5)
    model = _mine(_hf(0.1, 0.1, 0.1))
    st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2)
    mbs = [_cuda(pack_causal_lm_batch(_qa_padded(8, seed=60 + m), S, EOS)) for m in range(2)]
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


# ---------------------------------------------------------------------------------------- the Wenzhong-shaped recipe
def test_wenzhong_recipe_with_packing_collator_trains_checkpoints_and_resumes(launched, tmp_path):  # noqa: F811
    """finetune_wenzhong.py's structure (GPT2LMHeadModel.from_pretrained, GPT2QADataModel's dataset) with
    PackingCollator(default_collate, ...) and a training_step that also passes position_ids / segment_ids; dropout 0.1."""
    import argparse
    import hf_fixtures as F
    import pytorch_lightning as pl
    from pytorch_lightning import Trainer
    from pytorch_lightning.callbacks import ModelCheckpoint
    from torch.utils.data import DataLoader, default_collate
    from transformers import GPT2Config, GPT2LMHeadModel
    from fengshen.data.task_dataloader.medicalQADataset import GPT2QADataModel
    from fsb200.packing import PackingCollator
    mdir = tmp_path / "m"
    F.gpt2_tokenizer_dir(mdir)
    os.makedirs(tmp_path / "data")
    qa = [{"Question": f"q{i % 7}?" + "x" * (i % 5), "answer": f" rest {i % 3}." + "z" * (i % 11)} for i in range(48)]
    for name in ("train.txt", "valid.txt", "test.txt"):     # rows of 10 to 25 bytes: several fit one row of 64
        with open(tmp_path / "data" / name, "w", encoding="utf8") as f:
            f.writelines(repr(r) + "\n" for r in qa)
    cfg = {k: v for k, v in F.GPT2_CFG.items() if k != "model_type"}
    cfg.update(resid_pdrop=0.1, embd_pdrop=0.1, attn_pdrop=0.1)
    GPT2LMHeadModel(GPT2Config(**cfg)).save_pretrained(str(mdir))
    seen = []

    class Collator(PackingCollator):
        def __call__(self, samples):
            out = super().__call__(samples)
            seen.append(out)
            return out

    class GPT2FinetuneMedicalQA(pl.LightningModule):
        def __init__(self, args):
            super().__init__()
            self.args = args
            self.model = GPT2LMHeadModel.from_pretrained(args.pretrained_model_path)

        def training_step(self, batch, batch_idx):
            output = self.model(input_ids=batch['input_ids'], attention_mask=batch['attention_mask'],
                                labels=batch['labels'], position_ids=batch['position_ids'],
                                segment_ids=batch['segment_ids'])
            self.log('train_loss', output.loss)
            return output.loss

        def configure_optimizers(self):
            return torch.optim.AdamW(self.parameters(), lr=self.args.learning_rate)

    def fit(max_steps, resume):
        p = argparse.ArgumentParser("QA Task")
        p.add_argument('--do_eval_only', action='store_true', default=False)
        p.add_argument('--pretrained_model_path', type=str)
        p.add_argument('--learning_rate', default=1e-3, type=float)
        p = GPT2QADataModel.add_data_specific_args(p)
        p = Trainer.add_argparse_args(p)
        args = p.parse_args(["--pretrained_model_path", str(mdir), "--data_dir", str(tmp_path / "data"),
                             "--train_batchsize", "8", "--valid_batchsize", "8", "--max_seq_length", "64",
                             "--num_workers", "0", "--max_steps", str(max_steps), "--max_epochs", "-1", "--gpus", "1",
                             "--log_every_n_steps", "1", "--default_root_dir", str(tmp_path)])
        dm = GPT2QADataModel(args)
        module = GPT2FinetuneMedicalQA(args)
        ckpt = ModelCheckpoint(dirpath=str(tmp_path / "ckpt"), every_n_train_steps=3, save_last=True)
        trainer = Trainer.from_argparse_args(args, callbacks=[ckpt])
        ds = dm.train_data
        loader = DataLoader(ds, batch_size=args.train_batchsize, shuffle=True, num_workers=0,
                            collate_fn=Collator(default_collate, args.max_seq_length, ds.tokenizer.pad_token_id))
        trainer.fit(module, train_dataloaders=loader,
                    ckpt_path=str(tmp_path / "ckpt" / "last.ckpt") if resume else None)
        return trainer, module

    trainer, module = fit(6, False)
    m = module.model
    assert type(m).__module__ == "fsb200.hf" and m.p_attn == 0.1
    assert trainer.global_step == 6
    assert any(b["input_ids"].shape[0] < 8 for b in seen)           # samples shared rows
    assert (tmp_path / "ckpt" / "last.ckpt" / "checkpoint" / "mp_rank_00_model_states.pt").exists()
    w_before = m.flat.params.clone()
    trainer2, module2 = fit(8, True)
    assert trainer2.global_step == 8
    assert not torch.equal(module2.model.flat.params, w_before)
