"""GPU: mT5 / Randeng-T5 on packed batches (fsb200/packing.py pack_seq2seq_batch + MT5ForConditionalGeneration.forward(
segment_ids=..., decoder_segment_ids=...)), with dropout.

Parity: every packed sample run alone in transformers' MT5ForConditionalGeneration (fp32, CPU), at dropout 0 and at 0.1 with
F.dropout replayed from that sample's sub-blocks of the packed rows' masks (rebuilt by tests/philox_ref.py); the packed loss is
the target-weighted mean of the samples' losses. At dropout 0 the packed batch is the padded batch it came from, both bias
tables included in the gradient check. Exact: one full-length sample per row is the unpacked path at dropout 0 and 0.1;
no-grad equals grad; the CUDA-graph step equals eager under ZeRO-1 / ZeRO-2 with GA 2 at dropout 0.1; a batch without
labelled targets gives loss 0 and zero gradients. Also the per-launch fp64 and write-footprint censuses of a packed dropout
step, with this file's checkers for the packed attention forms."""
import math
import os
import random
import sys

import numpy as np
import pytest
import torch

import philox_ref as R
from test_t5_dropout_cpu import site_table
from test_t5_dropout_gpu import CFG, _hf, _mine

from fsb200.engine import ZeroEngine
from fsb200.packing import pack_seq2seq_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

PAD = 0
SE, SD = 128, 64        # packed row lengths (different, so a dropout site's shape names its side)


def _padded(n, seed, max_src=SE // 2, max_tgt=SD // 2, le=SE, ld=SD):
    """n samples in LCSTSDataset's format: source padded with the pad id under attention_mask 0, target labels -100 on the
    pads (some samples have no labelled target, one has a pad id labelled inside its target, as TaskT5Dataset does)."""
    rng = random.Random(seed)
    ids = torch.full((n, le), PAD, dtype=torch.int64)
    mask = torch.zeros((n, le), dtype=torch.int64)
    labels = torch.full((n, ld), -100, dtype=torch.int64)
    for i in range(n):
        ns, nt = rng.randint(3, max_src), rng.randint(0 if i == 3 else 2, max_tgt)
        ids[i, :ns] = torch.tensor([rng.randrange(2, CFG["vocab_size"]) for _ in range(ns)])
        mask[i, :ns] = 1
        if nt:
            labels[i, :nt] = torch.tensor([rng.randrange(2, CFG["vocab_size"]) for _ in range(nt)])
        if i == 1 and nt > 2:
            labels[i, 1] = PAD
    return {"input_ids": ids, "attention_mask": mask, "labels": labels}


def _samples(packed):
    """(row, enc start, enc end, dec start, dec end) of every sample of a packed batch (the pad tails left out)."""
    out = []
    for r in range(packed["input_ids"].shape[0]):
        e, d = packed["segment_ids"][r], packed["decoder_segment_ids"][r]
        m = int(e.max())
        for k in range(m + 1):
            es, ds = (e == k).nonzero().flatten(), (d == k).nonzero().flatten()
            if len(es) and len(ds) and (packed["labels"][r, ds] != -100).any():
                out.append((r, int(es[0]), int(es[-1]) + 1, int(ds[0]), int(ds[-1]) + 1))
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


@pytest.mark.parametrize("rate", [0.0, 0.1])
def test_packed_parity_with_transformers(rate, monkeypatch):
    torch.manual_seed(1)
    ref = _hf(rate)
    mine = _mine(ref)
    packed = pack_seq2seq_batch(_padded(10, seed=1), SE, SD, PAD)
    B = packed["input_ids"].shape[0]
    assert B < 10
    samples = _samples(packed)
    sites = site_table(CFG["num_layers"], CFG["num_decoder_layers"], B, SE, SD, CFG["d_model"], CFG["num_heads"],
                       CFG["d_ff"])
    seed = mine.dropout_seed
    full = {}
    if rate > 0:
        full = {site: (R.hidden_keep(seed, site, shape[0] * shape[1], shape[2], rate).reshape(shape) if kind == "hidden"
                       else R.attn_keep(seed, site, *shape, rate)) for site, kind, shape in sites}
    total, n_all, logits_ref = 0.0, 0, []
    for r, es, ee, ds, de in samples:
        span = {SE: slice(es, ee), SD: slice(ds, de)}
        calls = []

        def replay(x, p=0.5, training=True, inplace=False):
            site, kind, shape = sites[len(calls)]
            calls.append(site)
            if p == 0.0:
                return x
            keep = full[site][r:r + 1, span[shape[1]]] if kind == "hidden" else \
                full[site][r:r + 1, :, span[shape[2]], span[shape[3]]]
            assert tuple(keep.shape) == tuple(x.shape), (site, keep.shape, x.shape)
            return x * torch.from_numpy(np.ascontiguousarray(keep)).to(x.dtype) / (1.0 - p)
        monkeypatch.setattr(torch.nn.functional, "dropout", replay)
        lab = packed["labels"][r:r + 1, ds:de]
        out = ref(input_ids=packed["input_ids"][r:r + 1, es:ee], labels=lab)
        monkeypatch.undo()
        assert len(calls) == len(sites)
        n = int((lab != -100).sum())
        total, n_all = total + out.loss * n, n_all + n
        logits_ref.append(out.logits.detach()[0])
    loss_ref = total / n_all
    loss_ref.backward()
    out, g = _run(mine, packed, return_logits=True)
    assert abs(out.loss.item() - loss_ref.item()) <= 3e-3 + 5e-4 * abs(loss_ref.item()), (out.loss.item(), loss_ref.item())
    lg = out.logits.float().cpu()
    for (r, es, ee, ds, de), want in zip(samples, logits_ref):
        assert (lg[r, ds:de] - want).abs().max().item() <= 4 * 2.0 ** -8 * want.abs().max().item(), (r, ds, de)
    refp = dict(ref.named_parameters())
    for name, got in g.items():
        want = refp[name].grad.flatten()
        assert _cos(got, want) >= 0.998, name
        assert abs(got.norm().item() / (want.norm().item() + 1e-30) - 1.0) <= 0.03, name
    assert len(g) == len(refp)


def test_dropout_zero_packed_matches_padded():
    mine = _mine(_hf(0.0))
    padded = _padded(10, seed=2)
    packed = pack_seq2seq_batch(padded, SE, SD, PAD)
    o_p, g_p = _run(mine, packed)
    o_d, g_d = _run(mine, padded)
    assert abs(o_p.loss.item() - o_d.loss.item()) <= 3e-3, (o_p.loss.item(), o_d.loss.item())
    for name in g_p:
        assert _cos(g_p[name], g_d[name]) >= 0.999, name
    assert any("relative_attention_bias" in n for n in g_p if n.startswith("encoder"))
    assert any("relative_attention_bias" in n for n in g_p if n.startswith("decoder"))


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_one_full_sample_per_row_is_the_unpacked_path_bit_for_bit(p):
    """Every source fills its row and every target its row: each side is one segment with the same id, so the packed forms
    run over exactly what the unpacked kernels do (and the decoder input is the same shifted labels)."""
    g = torch.Generator().manual_seed(5)
    batch = {"input_ids": torch.randint(2, CFG["vocab_size"], (2, SE), generator=g),
             "labels": torch.randint(2, CFG["vocab_size"], (2, SD), generator=g)}
    runs = []
    for packed in (False, True):
        torch.manual_seed(11)           # the dropout seed is drawn at construction
        m = _mine(_hf(p))
        kw = {} if not packed else {"segment_ids": torch.zeros(2, SE, dtype=torch.int64),
                                    "decoder_segment_ids": torch.zeros(2, SD, dtype=torch.int64)}
        out, gr = _run(m, batch, **kw)
        runs.append((out.loss.item(), gr))
    (l0, g0), (l1, g1) = runs
    assert l0 == l1
    assert all(torch.equal(g0[n], g1[n]) for n in g0)


def test_decoder_inputs_restart_at_every_segment():
    """Each decoder segment starts from the start id (the previous sample's last label is not its input): a packed row's
    logits for sample 2 do not change when sample 1's labels do."""
    mine = _mine(_hf(0.0))
    mine.eval()
    batch = {"input_ids": torch.randint(2, 500, (1, SE)), "segment_ids": torch.tensor([[0] * 60 + [1] * 68]),
             "labels": torch.randint(2, 500, (1, SD)), "decoder_segment_ids": torch.tensor([[0] * 20 + [1] * 44])}
    a = mine(**_cuda(batch), return_logits=True).logits
    changed = dict(batch, labels=batch["labels"].clone())
    changed["labels"][0, 19] = 1 + int(batch["labels"][0, 19]) % 400
    b = mine(**_cuda(changed), return_logits=True).logits
    assert torch.equal(a[0, 20:], b[0, 20:])


def test_packed_loss_curve_follows_the_padded_curve():
    curves = []
    for pack in (False, True):
        model = _mine(_hf(0.0))
        eng = ZeroEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1)
        curve = []
        for it in range(20):
            padded = _padded(8, seed=100 + it % 4)
            out = model(**_cuda(pack_seq2seq_batch(padded, SE, SD, PAD) if pack else padded))
            out.loss.backward()
            eng.backward_done()
            eng.step(lr=1e-3)
            curve.append(out.loss.item())
        curves.append(curve)
    a, b = np.array(curves[0]), np.array(curves[1])
    assert bool((np.abs(a - b) <= 1e-2 + 1e-3 * np.abs(a)).all()), curves     # the test model's losses start near 130


def test_no_grad_loss_equals_grad_loss_with_dropout():
    model = _mine(_hf(0.1))
    batch = _cuda(pack_seq2seq_batch(_padded(8, seed=3), SE, SD, PAD))
    with torch.no_grad():
        l0 = model(**batch).loss.item()
    model.dropout_counter.zero_()
    out = model(**batch)
    assert out.loss.item() == l0
    out.loss.backward()


def test_batch_without_targets_gives_zero_loss_and_gradients():
    """Every sample's target is empty: the packer emits one all-pad row with every label ignored, and the cross-entropy
    (which divides by max(labelled targets, 1)) gives exactly 0, so every gradient is exactly 0."""
    padded = _padded(4, seed=6)
    padded["labels"][:] = -100
    packed = pack_seq2seq_batch(padded, SE, SD, PAD)
    assert packed["input_ids"].shape[0] == 1 and bool((packed["labels"] == -100).all())
    model = _mine(_hf(0.1))
    out, g = _run(model, packed)
    assert out.loss.item() == 0.0
    assert all(bool((t == 0).all()) for t in g.values())


@pytest.mark.parametrize("stage", [1, 2])
def test_cuda_graph_step_equals_eager_on_packed_batches_with_dropout(stage):
    """Fixed-shape packed micro-batches [2, SE] / [2, SD] (the segment ids are two more static batch buffers), GA 2,
    dropout 0.1."""
    from fsb200.trainer import PretrainStep
    runs = []
    for graph in (False, True):
        torch.manual_seed(3)
        model = _mine(_hf(0.1))
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2,
                          stage=stage, cuda_graph=graph)
        losses = []
        for it in range(4):
            mbs = []
            for m in range(2):
                p = pack_seq2seq_batch(_padded(16, seed=300 + 2 * it + m), SE, SD, PAD)
                assert p["input_ids"].shape[0] >= 2
                mbs.append({k: v[:2].cuda() for k, v in p.items() if k != "attention_mask"})
            losses.append(float(st.step_device(mbs)))
        runs.append((losses, model.flat.params.clone(), int(model.dropout_counter.item())))
    (l0, p0, c0), (l1, p1, c1) = runs
    assert c0 == c1 == 4 * 2 * model.dropout_sites
    assert l0 == l1, (l0, l1)
    assert torch.equal(p0, p1)


def test_refusals():
    model = _mine(_hf(0.1))
    packed = pack_seq2seq_batch(_padded(6, seed=4), SE, SD, PAD)
    with pytest.raises(ValueError, match="together"):
        model(**{k: v.cuda() for k, v in packed.items() if k != "decoder_segment_ids"})
    with pytest.raises(ValueError, match="together"):
        model(**{k: v.cuda() for k, v in packed.items() if k != "segment_ids"})
    bad = packed["attention_mask"].clone()
    bad[0, -1] = 0
    with pytest.raises(ValueError, match="attention_mask has zeros"):
        model(**dict(_cuda(packed), attention_mask=bad))          # a host mask: checked exactly
    ids = packed["segment_ids"].clone()
    ids[0, 0] = 5
    with pytest.raises(ValueError, match="non-decreasing"):                   # host ids: checked exactly
        model(**dict(_cuda(packed), segment_ids=ids, decoder_segment_ids=packed["decoder_segment_ids"]))
    from fsb200.models.t5 import MT5ForConditionalGeneration
    import copy
    cfg = copy.copy(_hf(0.0).config)
    cfg.d_kv = 128
    m128 = MT5ForConditionalGeneration(cfg, device="cuda")
    with pytest.raises(ValueError, match="d_kv 64"):
        m128(**_cuda(packed))
    out = model(**_cuda(packed))
    assert math.isfinite(out.loss.item())


# ---------------------------------------------------------------------------------------- per-launch censuses
def _ref_attention(q, k, v, scale, vis, rel, drop_mult):
    """fp64 O of one row [H, Sq, D] under vis [Sq, Skv] with the bias vector rel [H, Sq + Skv - 1] (or None)."""
    qf, kf, vf = (t.double().permute(1, 0, 2).detach().requires_grad_(True) for t in (q, k, v))
    s = scale * qf @ kf.transpose(-1, -2)
    relf = None
    if rel is not None:
        relf = rel.double().detach().requires_grad_(True)
        Sq, Skv = q.shape[0], k.shape[0]
        idx = torch.arange(Skv, device=q.device)[None, :] - torch.arange(Sq, device=q.device)[:, None] + Sq - 1
        s = s + relf[:, idx]
    has = vis.any(-1)[None, :, None]
    s = s.masked_fill(~vis[None], float("-inf")).masked_fill(~has, 0.0)
    o = (torch.softmax(s, -1) * has * drop_mult) @ vf
    return o, torch.logsumexp(s, -1), has[..., 0], (qf, kf, vf, relf)


def _vis(b, seg_start, seg_end, causal, kv_bounds, Skv):
    k = torch.arange(Skv, device=seg_start.device)
    v = (k[None, :] >= seg_start[b].long()[:, None]) & (k[None, :] < seg_end[b].long()[:, None])
    if causal and kv_bounds is None:
        v = v & (k[None, :] <= torch.arange(seg_start.shape[1], device=v.device)[:, None])
    return v


def _mult(drop, b, H, Sq, Skv, dev):
    import launch_refs as LR
    return LR.attn_mult(LR.drop_spec(drop), range(b, b + 1), H, Sq, Skv, dev)[0] if drop is not None else 1.0


def check_sdpa_segments_fwd(real, bound, q, k, v, scale, seg_start, seg_end, out=None, drop=None, causal=True,
                            rel_bias=None, kv_bounds=None):
    """Every segment form against fp64, row by row (the dropout keep mask is at the row-relative (q, k))."""
    o, lse = ret = real(q, k, v, scale, seg_start, seg_end, out=out, drop=drop, causal=causal, rel_bias=rel_bias,
                        kv_bounds=kv_bounds)
    H = q.shape[2]
    for b in range(q.shape[0]):
        vis = _vis(b, seg_start, seg_end, causal, kv_bounds, k.shape[1])
        ref, s, has, _ = _ref_attention(q[b], k[b], v[b], scale, vis, rel_bias, _mult(drop, b, H, q.shape[1], k.shape[1],
                                                                                       q.device))
        bound.close("O", o[b].permute(1, 0, 2), ref.detach(), 2e-2 * max(1.0, ref.abs().max().item() / 4))
        lg = (lse[b].double() * math.log(2.0)).masked_fill(~has, 0.0)
        bound.close("lse", lg, s.detach().masked_fill(~has, 0.0), 2e-3)
    return ret


def check_sdpa_segments_bwd(real, bound, q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv, drop=None,
                            causal=True, rel_bias=None, drel_bias=None, kv_bounds=None):
    """Gradients against fp64 row by row; drel_bias is accumulated into (+=): its increment is checked against the sum of
    the rows' fp64 bias gradients."""
    before = None if drel_bias is None else drel_bias.clone()
    ret = real(q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv, drop=drop, causal=causal, rel_bias=rel_bias,
               drel_bias=drel_bias, kv_bounds=kv_bounds)
    H = q.shape[2]
    drel_ref = 0.0
    for b in range(q.shape[0]):
        vis = _vis(b, seg_start, seg_end, causal, kv_bounds, k.shape[1])
        with torch.enable_grad():     # the step's backward runs with autograd recording off
            ref, _, _, (qf, kf, vf, relf) = _ref_attention(q[b], k[b], v[b], scale, vis, rel_bias,
                                                          _mult(drop, b, H, q.shape[1], k.shape[1], q.device))
            ref.backward(dout[b].double().permute(1, 0, 2))
        for name, got, want in (("dQ", dq, qf.grad), ("dK", dk, kf.grad), ("dV", dv, vf.grad)):
            bound.close(name, got[b].permute(1, 0, 2), want, 3e-2 * max(1.0, want.abs().max().item()))
        if drel_bias is not None:
            drel_ref = drel_ref + relf.grad
    if drel_bias is not None:
        want = drel_ref
        bound.close("dRel", drel_bias.double() - before.double(), want, 2e-2 * max(1.0, want.abs().max().item()))
    return ret


def _packed_dropout_census(monkeypatch, checkers):
    """One packed mT5 training step at dropout 0.1, GA 2, every op launch recorded and its first call of each signature
    checked by `checkers`; returns the recorder."""
    from launch_census import Recorder
    from fsb200 import lib as L
    from fsb200.trainer import PretrainStep
    torch.manual_seed(5)
    model = _mine(_hf(0.1))
    st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2)
    mbs = [_cuda(pack_seq2seq_batch(_padded(10, seed=60 + m), SE, SD, PAD)) for m in range(2)]
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
        for form in (("rel_bias", "T"), ("kv_bounds", "tuple")):
            assert any(k[0] == op and any(x[0] == form[0] and x[1] is not None for x in k[1]) for k in rec.checked), \
                f"no {op} with {form[0]} was checked"
    assert L.launch_count - c0 - rec.extra_launches == rec.wrapped_launches
    assert math.isfinite(float(loss.item()))
    return rec


def test_every_launch_of_a_packed_dropout_step_against_fp64(monkeypatch):
    import launch_refs as LR
    import test_llama_packing_gpu as LP
    checkers = dict(LR.CHECKERS)
    checkers.update(segment_bounds=LP.check_segment_bounds, sdpa_segments_fwd=check_sdpa_segments_fwd,
                    sdpa_segments_bwd=check_sdpa_segments_bwd)
    # this step's gradients have denormal entries (unscaled T5 attention on the test model's std-1 embeddings), where
    # check_adamw_flat's relative bound is below fp32 resolution; the optimizer runs unchecked here and is checked by the
    # other censuses
    checkers["adamw_flat"] = lambda real, bound, *a, **k: real(*a, **k)
    _packed_dropout_census(monkeypatch, checkers)


def test_write_footprint_of_every_launch_of_a_packed_dropout_step(monkeypatch):
    """With a bias, sdpa_segments_bwd also accumulates into drel_bias, as sdpa_bwd does: the same write contract."""
    import footprint as F
    monkeypatch.setitem(F.WRITES, "sdpa_segments_bwd", F._sdpa_bwd)
    stats = F.Stats()
    _packed_dropout_census(monkeypatch, F.footprint_checkers(stats))
    assert {"sdpa_segments_fwd", "sdpa_segments_bwd"} <= set(stats.checked)


# ---------------------------------------------------------------------------------------- the mt5_summary-shaped recipe
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


def _lcsts_item(text, summary, max_enc, max_dec):
    """An item in the format of LCSTSDataset.encode (tests/golden/t5_finetune_batches.npz pins it on the reference):
    one id per character, eos 1, pad 0; the summary's pad ids stay labelled, as the reference leaves them."""
    enc = [2 + ord(c) % 500 for c in text][:max_enc - 1] + [1]
    dec = [2 + ord(c) % 500 for c in summary][:max_dec - 1] + [1]
    return {"input_ids": torch.tensor(enc + [0] * (max_enc - len(enc))),
            "attention_mask": torch.tensor([1] * len(enc) + [0] * (max_enc - len(enc))),
            "labels": torch.tensor(dec + [0] * (max_dec - len(dec))), "text": text, "summary": summary}


def test_mt5_summary_recipe_with_packing_collator_trains_checkpoints_and_resumes(launched, tmp_path):
    """mt5_summary.py's structure (MT5ForConditionalGeneration.from_pretrained, items in LCSTSDataset.encode's format) with Seq2SeqPackingCollator(default_collate, ...) and a training_step that also passes the packed
    segment ids; dropout 0.1, through Trainer.fit, checkpoint and resume."""
    import argparse
    import hf_fixtures as F
    import pytorch_lightning as pl
    from pytorch_lightning import Trainer
    from pytorch_lightning.callbacks import ModelCheckpoint
    from torch.utils.data import DataLoader, default_collate
    from transformers import MT5Config, MT5ForConditionalGeneration
    from fsb200.packing import Seq2SeqPackingCollator
    mdir = tmp_path / "m"
    cfg = {k: v for k, v in F.MT5_CFG.items() if k != "model_type"}
    cfg.update(dropout_rate=0.1)
    MT5ForConditionalGeneration(MT5Config(**cfg)).save_pretrained(str(mdir))
    rng = random.Random(0)
    items = [_lcsts_item("t" * rng.randint(3, 50), "s" * rng.randint(0, 20), 64, 16) for _ in range(48)]
    seen = []

    class Collator(Seq2SeqPackingCollator):
        def __call__(self, samples):
            out = super().__call__(samples)
            seen.append(out)
            return out

    class MT5FinetuneSummary(pl.LightningModule):
        def __init__(self, args):
            super().__init__()
            self.args = args
            self.model = MT5ForConditionalGeneration.from_pretrained(args.pretrained_model_path)

        def training_step(self, batch, batch_idx):
            output = self.model(input_ids=batch['input_ids'], attention_mask=batch['attention_mask'],
                                labels=batch['labels'], segment_ids=batch['segment_ids'],
                                decoder_segment_ids=batch['decoder_segment_ids'])
            self.log('train_loss', output.loss)
            return output.loss

        def configure_optimizers(self):
            return torch.optim.AdamW(self.parameters(), lr=self.args.learning_rate)

    def fit(max_steps, resume):
        p = argparse.ArgumentParser("Summary Task")
        p.add_argument('--pretrained_model_path', type=str)
        p.add_argument('--learning_rate', default=1e-3, type=float)
        p = Trainer.add_argparse_args(p)
        args = p.parse_args(["--pretrained_model_path", str(mdir), "--max_steps", str(max_steps), "--max_epochs", "-1",
                             "--gpus", "1", "--log_every_n_steps", "1", "--default_root_dir", str(tmp_path)])
        module = MT5FinetuneSummary(args)
        ckpt = ModelCheckpoint(dirpath=str(tmp_path / "ckpt"), every_n_train_steps=3, save_last=True)
        trainer = Trainer.from_argparse_args(args, callbacks=[ckpt])
        # rows twice the padded lengths: LCSTSDataset labels its target pads, so targets keep their full 16 tokens
        loader = DataLoader(items, batch_size=8, shuffle=True, num_workers=0,
                            collate_fn=Collator(default_collate, 2 * 64, 2 * 16, 0))
        trainer.fit(module, train_dataloaders=loader,
                    ckpt_path=str(tmp_path / "ckpt" / "last.ckpt") if resume else None)
        return trainer, module

    trainer, module = fit(6, False)
    m = module.model
    assert type(m).__module__ == "fsb200.hf" and m.p_drop == 0.1 and int(m.dropout_counter.item()) > 0
    assert trainer.global_step == 6
    assert all(b["input_ids"].shape[0] == 4 for b in seen)          # two samples per row
    assert (tmp_path / "ckpt" / "last.ckpt" / "checkpoint" / "mp_rank_00_model_states.pt").exists()
    w_before = m.flat.params.clone()
    trainer2, module2 = fit(8, True)
    assert trainer2.global_step == 8
    assert not torch.equal(module2.model.flat.params, w_before)
