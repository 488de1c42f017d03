"""GPU: Ziya-LLaMA on packed batches (fsb200/packing.py + LlamaForCausalLM.forward(segment_ids=...)).

A packed batch holds the same labelled targets as the padded batch it came from, each predicted from the same context, so
its loss and gradients are those of the padded batch: checked against the fp32 oracle (oracle/llama_oracle.py) on the padded
batch at the DESIGN §4 bars (loss |delta| <= 3e-3, per-parameter gradient cosine >= 0.999) and against fsb200's own padded
step, and each packed sample's logits are those of the sample run alone. Exact: all-zero segment_ids is the unsegmented path
bit for bit; the model ignores segment-start labels by itself; the CUDA-graph step is the eager step bit for bit. Also: int8 /
int4 no-grad forwards, a batch without labels, the per-launch fp64 census of a packed step, tensor parallelism (2 GPUs) and
the Ziya-shaped example script through Trainer.fit with PackingCollator, checkpoint and resume."""
import glob
import math
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import llama_oracle as O  # noqa: E402  (checker only)

from fsb200.engine import ZeroEngine  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402
from fsb200.packing import pack_causal_lm_batch  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "llama_*.npz")))
EOS = 2


def _cfg(V, h, L, nh):
    return SimpleNamespace(vocab_size=V, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                           rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                           llama_mlp_multiple_of=256)


def _build(path, **kw):
    g = np.load(path)
    V, h, L, nh, _, S = (int(x) for x in g["config"])
    sd = O.make_weights(V, h, L, seed=int(g["weight_seed"]))
    model = LlamaForCausalLM(_cfg(V, h, L, nh), device="cuda", **kw)
    model.load_reference_state_dict(sd)
    return model, sd, V, nh, S


def _sft_padded(V, n, max_len, seed):
    """n SFT-like samples (prompt with label -100, then the labelled output), eos-padded to the longest: the format of the
    Ziya SFT collator (examples/ziya_llama/finetune_ziya_llama.py:36-85)."""
    rng = random.Random(seed)
    ids, labs = [], []
    for _ in range(n):
        p = [rng.randrange(3, V) for _ in range(rng.randint(1, max_len // 4))]
        o = [rng.randrange(3, V) for _ in range(rng.randint(1, max_len // 3))] + [EOS]
        ids.append(p + o)
        labs.append([-100] * len(p) + o)
    L = max(len(i) for i in ids)
    return {"input_ids": torch.tensor([i + [EOS] * (L - len(i)) for i in ids]),
            "labels": torch.tensor([l + [-100] * (L - len(l)) for l in labs]),
            "position_ids": torch.arange(L)[None].expand(n, L).contiguous()}


def _grads(model):
    return {n: p.main_grad.float().cpu().flatten().clone() for n, p in model.named_parameters()}


def _cos(a, b):
    return (torch.dot(a, b) / (a.norm() * b.norm() + 1e-30)).item()


def _run(model, batch):
    model.flat.grads.zero_()
    out = model(**{k: v.cuda() for k, v in batch.items()})
    out.loss.backward()
    torch.cuda.synchronize()
    return out.loss.item(), _grads(model)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_packed_matches_oracle_and_padded(path):
    model, sd, V, nh, S = _build(path)
    padded = _sft_padded(V, 7, S, seed=1)
    packed = pack_causal_lm_batch(padded, S, EOS)
    assert packed["input_ids"].shape[0] < 7       # the samples really share rows
    loss_p, g_p = _run(model, packed)
    loss_d, g_d = _run(model, {k: padded[k] for k in ("input_ids", "labels", "position_ids")})
    osd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    oloss, _ = O.forward(osd, padded, nh)
    oloss.backward()
    assert abs(loss_p - oloss.item()) <= 3e-3, (loss_p, oloss.item())
    assert abs(loss_p - loss_d) <= 3e-3, (loss_p, loss_d)
    for name in g_p:
        assert _cos(g_p[name], osd[name].grad.flatten()) >= 0.999, name
        assert _cos(g_p[name], g_d[name]) >= 0.999, name


def test_zero_segment_ids_is_the_unsegmented_path_bit_for_bit():
    model, sd, V, nh, S = _build(GOLDEN[0])
    b = O.make_batch(V, 2, S, seed=5)
    batch = {k: b[k] for k in ("input_ids", "labels", "position_ids")}
    loss0, g0 = _run(model, batch)
    loss1, g1 = _run(model, dict(batch, segment_ids=torch.zeros_like(b["input_ids"])))
    assert loss0 == loss1
    assert all(torch.equal(g0[n], g1[n]) for n in g0)


def test_packed_loss_curve_follows_the_padded_curve():
    curves = []
    for pack in (False, True):
        model, sd, V, nh, S = _build(GOLDEN[0])
        eng = ZeroEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1)
        curve = []
        for it in range(20):
            padded = _sft_padded(V, 6, S, seed=100 + it % 4)
            batch = pack_causal_lm_batch(padded, S, EOS) if pack else padded
            out = model(**{k: v.cuda() for k, v in batch.items()})
            out.loss.backward()
            eng.backward_done()
            eng.step(lr=1e-3)
            curve.append(out.loss.item())
        curves.append(curve)
    err = np.abs(np.array(curves[0]) - np.array(curves[1])).max()
    assert err <= 1e-2, (err, curves)


def test_no_grad_loss_equals_grad_loss():
    model, sd, V, nh, S = _build(GOLDEN[1])
    batch = {k: v.cuda() for k, v in pack_causal_lm_batch(_sft_padded(V, 6, S, seed=3), S, EOS).items()}
    with torch.no_grad():
        l0 = model(**batch).loss.item()
    out = model(**batch)
    assert out.loss.item() == l0
    out.loss.backward()


@pytest.mark.parametrize("stage", [1, 2])
def test_cuda_graph_step_equals_eager_on_packed_batches(stage):
    """Fixed-shape packed micro-batches (segment_ids is one more static batch buffer), gradient accumulation 2."""
    from fsb200.trainer import PretrainStep
    runs = []
    for graph in (False, True):
        model, sd, V, nh, S = _build(GOLDEN[0])
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2,
                          stage=stage, cuda_graph=graph)
        losses = []
        for it in range(4):
            mbs = []
            for m in range(2):
                p = pack_causal_lm_batch(_sft_padded(V, 10, S, seed=300 + 2 * it + m), S, EOS)
                mbs.append({k: v[:2].cuda() for k, v in p.items() if k != "attention_mask"})   # fixed [2, S]
            losses.append(float(st.step_device(mbs)))
        runs.append((losses, model.flat.params.clone()))
    (l0, p0), (l1, p1) = runs
    assert l0 == l1, (l0, l1)
    assert torch.equal(p0, p1)


def test_fp8_trains_on_packed_batches():
    model, sd, V, nh, S = _build(GOLDEN[1], fp8=True)
    padded = _sft_padded(V, 6, S, seed=8)
    packed = pack_causal_lm_batch(padded, S, EOS)
    loss, _ = _run(model, packed)
    oloss, _ = O.forward(sd, padded, nh)
    assert abs(loss - oloss.item()) <= 1e-2, (loss, oloss.item())   # FP8 projections: the FP8 tests' loss bar


def test_model_ignores_segment_start_labels_itself():
    """The packer already sets segment-start labels to -100; the model must do it on its own too: labels left on the starts
    give the loss and gradients of the batch with the starts masked by hand, bit for bit."""
    model, sd, V, nh, S = _build(GOLDEN[0])
    packed = pack_causal_lm_batch(_sft_padded(V, 7, S, seed=21), S, EOS)
    raw = dict(packed, labels=packed["labels"].clone())
    seg = packed["segment_ids"]
    starts = torch.ones_like(seg, dtype=torch.bool)
    starts[:, 1:] = seg[:, 1:] != seg[:, :-1]
    raw["labels"][starts] = packed["input_ids"][starts]       # a (wrong) target on every segment start
    assert (raw["labels"] != packed["labels"]).any()
    l0, g0 = _run(model, packed)
    l1, g1 = _run(model, raw)
    assert l0 == l1
    assert all(torch.equal(g0[n], g1[n]) for n in g0)


@pytest.mark.parametrize("path", GOLDEN[:2], ids=[os.path.basename(p) for p in GOLDEN[:2]])
def test_each_packed_sample_sees_only_itself(path):
    """Every sample's logits in the packed rows equal its logits run alone (batch 1, its own length), within bf16 noise."""
    model, sd, V, nh, S = _build(path)
    packed = pack_causal_lm_batch(_sft_padded(V, 7, S, seed=4), S, EOS)
    with torch.no_grad():
        lg = model(**{k: v.cuda() for k, v in packed.items()}, return_logits=True).logits.float()
        seg = packed["segment_ids"]
        checked = 0
        for r in range(seg.shape[0]):
            row = seg[r].tolist()
            s = 0
            for t in range(1, S + 1):
                if t == S or row[t] != row[t - 1]:
                    if not (packed["labels"][r, s:t] == -100).all():      # a sample (not the pad tail)
                        ids = packed["input_ids"][r:r + 1, s:t].cuda()
                        alone = model(input_ids=ids, position_ids=torch.arange(t - s)[None].cuda(),
                                      return_logits=True).logits.float()
                        want, got = alone[0], lg[r, s:t]
                        tol = 4 * 2.0 ** -8 * want.abs().max().item()
                        assert (got - want).abs().max().item() <= tol, (r, s, t)
                        checked += 1
                    s = t
        assert checked >= 7


def test_batch_without_labels_gives_zero_loss_and_gradients():
    """pack_causal_lm_batch turns a batch with no labelled token into one all-pad row with every label ignored: the fused
    cross-entropy divides by max(n_valid, 1), so the loss and every gradient are exactly 0."""
    model, sd, V, nh, S = _build(GOLDEN[0])
    empty = pack_causal_lm_batch({"input_ids": torch.full((2, 8), 5), "labels": torch.full((2, 8), -100)}, S, EOS)
    assert empty["input_ids"].shape == (1, S)
    loss, g = _run(model, empty)
    assert loss == 0.0
    assert all(not v.any() for v in g.values())


@pytest.mark.parametrize("fmt", ["load_in_8bit", "load_in_4bit"])
def test_quantized_no_grad_forward_on_packed_batches(fmt):
    """int8 / int4 models (inference only) run the packed no-grad forward: the loss of the padded batch, and every sample's
    logits as in the padded batch."""
    g = np.load(GOLDEN[1])
    V, h, L, nh, _, S = (int(x) for x in g["config"])
    sd = O.make_weights(V, h, L, seed=int(g["weight_seed"]))
    model = LlamaForCausalLM(_cfg(V, h, L, nh), device="cuda", **{fmt: True})
    model.load_reference_state_dict(sd)
    padded = _sft_padded(V, 6, S, seed=9)
    packed = pack_causal_lm_batch(padded, S, EOS)
    with torch.no_grad():
        lp = model(**{k: v.cuda() for k, v in packed.items()}).loss.item()
        ld = model(**{k: v.cuda() for k, v in padded.items()}).loss.item()
    assert math.isfinite(lp) and abs(lp - ld) <= 3e-3, (lp, ld)


# ---------------------------------------------------------------------------------------- per-launch fp64 census
def _bounds_runs(seg_start, seg_end):
    """Per row the (start, end) runs of the bounds."""
    st, en = seg_start.cpu().tolist(), seg_end.cpu().tolist()
    out = []
    for a, b in zip(st, en):
        runs, t = [], 0
        while t < len(a):
            runs.append((a[t], b[t]))
            t = b[t]
        out.append(runs)
    return out


def check_segment_bounds(real, bound, segment_ids):
    st, en = real(segment_ids)
    want_s, want_e = torch.empty_like(st), torch.empty_like(en)
    for r, row in enumerate(segment_ids.cpu().tolist()):
        s = 0
        for t in range(1, len(row) + 1):
            if t == len(row) or row[t] != row[t - 1]:
                want_s[r, s:t], want_e[r, s:t] = s, t
                s = t
    assert torch.equal(st, want_s) and torch.equal(en, want_e), "segment_bounds differs from the plain restatement"
    return st, en


def check_sdpa_segments_fwd(real, bound, q, k, v, scale, seg_start, seg_end, out=None):
    """Each segment is a causal attention of its own: launch_refs' fp64 causal bounds on its slices."""
    import launch_refs as R
    o, lse = ret = real(q, k, v, scale, seg_start, seg_end, out=out)
    for b, runs in enumerate(_bounds_runs(seg_start, seg_end)):
        for s, e in runs:
            sl = lambda t: t[b:b + 1, s:e]
            R.verify_sdpa_fwd(bound, sl(q), sl(k), sl(v), scale, True, None, None, sl(o), lse[b:b + 1, :, s:e])
    return ret


def check_sdpa_segments_bwd(real, bound, q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv):
    import launch_refs as R
    ret = real(q, k, v, out, dout, lse, scale, seg_start, seg_end, dq, dk, dv)
    for b, runs in enumerate(_bounds_runs(seg_start, seg_end)):
        for s, e in runs:
            sl = lambda t: t[b:b + 1, s:e]
            R.verify_sdpa_bwd(bound, sl(q), sl(k), sl(v), sl(out), sl(dout), lse[b:b + 1, :, s:e], scale, True, sl(dq),
                              sl(dk), sl(dv))
    return ret


def test_every_launch_of_a_packed_step_against_fp64(monkeypatch):
    import launch_refs as R
    from launch_census import Recorder
    from fsb200 import lib as L
    from fsb200.trainer import PretrainStep
    checkers = dict(R.CHECKERS)
    checkers.update(segment_bounds=check_segment_bounds, sdpa_segments_fwd=check_sdpa_segments_fwd,
                    sdpa_segments_bwd=check_sdpa_segments_bwd)
    model, sd, V, nh, S = _build(GOLDEN[0])
    st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2)
    mbs = [{k: v.cuda() for k, v in pack_causal_lm_batch(_sft_padded(V, 7, S, seed=60 + m), S, EOS).items()}
           for m in range(2)]
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
    assert L.launch_count - c0 - rec.extra_launches == rec.wrapped_launches
    assert math.isfinite(float(loss.item()))


# ---------------------------------------------------------------------------------------- tensor parallelism
TP_V, TP_H, TP_NL, TP_NH, TP_S = 512, 256, 2, 4, 128


def _tp_run(rank, world, port, q):
    sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))
    import torch.distributed as dist
    from fengshen.utils.llama_convert import split_state_dict_tp
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    tp_group = None
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        tp_group = dist.new_group(list(range(world)))
    full = O.make_weights(TP_V, TP_H, TP_NL, seed=0)
    model = LlamaForCausalLM(_cfg(TP_V, TP_H, TP_NL, TP_NH), device=dev, world_size=1, tp_group=tp_group)
    model.load_reference_state_dict(split_state_dict_tp(full, world, TP_NH)[rank] if world > 1 else full)
    dp_group = None
    if world > 1:
        dp_group = [dist.new_group([r]) for r in range(world)][rank]
    eng = ZeroEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, process_group=dp_group,
                     tp_group=tp_group)
    losses, g0 = [], None
    for it in range(3):
        b = pack_causal_lm_batch(_sft_padded(TP_V, 8, TP_S, seed=70 + it), TP_S, EOS)
        out = model(**{k: v.to(dev) for k, v in b.items()})
        out.loss.backward()
        if it == 0:
            g0 = {n: p.main_grad.float().cpu().numpy().copy() for n, p in model.named_parameters()}
        eng.backward_done()
        eng.step()
        losses.append(out.loss.item())
    eng.wait_params()
    q.put((world, rank, losses, g0))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tensor_parallel_2_matches_single_gpu_on_packed_batches():
    sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))
    from fengshen.utils.llama_convert import merge_state_dict_tp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_run, args=(r, 2, 29863, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in range(2)), key=lambda r: r[1])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    p1 = ctx.Process(target=_tp_run, args=(0, 1, 0, q))
    p1.start()
    single = q.get(timeout=300)
    p1.join(timeout=60)
    assert res[0][2] == res[1][2]
    for a, b in zip(res[0][2], single[2]):
        assert abs(a - b) < 5e-3, (res[0][2], single[2])
    T = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
    merged = merge_state_dict_tp([T(res[0][3]), T(res[1][3])], TP_NH)
    for name, want in T(single[3]).items():
        assert _cos(merged[name].flatten(), want.flatten()) > 0.999, name


# ---------------------------------------------------------------------------------------- the Ziya-shaped script
class _SFTCollator:
    """LlamaSFTCollator's output format from the example's token rows: a prompt and an output of per-sample lengths,
    eos-padded to the longest, labels -100 on the prompt and the pads."""

    def __call__(self, samples):
        ids, labs = [], []
        for x in samples:
            x = x.tolist()
            n = 8 + sum(x) % 40
            p = 2 + x[0] % 5
            ids.append(x[:n])
            labs.append([-100] * p + x[p:n])
        L = max(len(i) for i in ids)
        return {"input_ids": torch.tensor([i + [EOS] * (L - len(i)) for i in ids]),
                "labels": torch.tensor([l + [-100] * (L - len(l)) for l in labs]),
                "attention_mask": torch.ones((len(ids), L)),
                "position_ids": torch.arange(L)[None].expand(len(ids), L).contiguous()}


def test_example_script_with_packing_collator_trains_checkpoints_and_resumes(tmp_path, monkeypatch):
    """examples/pretrain_ziya_llama.py (the structure of finetune_ziya_llama.py) with PackingCollator around an SFT-format
    collator: `self.model(**batch)` picks up segment_ids, Trainer.fit trains, checkpoints and resumes."""
    for p in (os.path.join(ROOT, "fengshen-lm_b200", "compat"), os.path.join(ROOT, "examples")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import pretrain_ziya_llama as ex
    from fsb200.packing import PackingCollator
    seen = []

    class Collator(PackingCollator):
        def __call__(self, samples):
            out = super().__call__(samples)
            seen.append(out)
            return out
    monkeypatch.setattr(ex, "SyntheticCollator", lambda: Collator(_SFTCollator(), 64, EOS))

    def args(extra=()):
        return ["--hidden_size", "256", "--num_layers", "2", "--num_heads", "4", "--vocab_size", "512",
                "--max_seq_length", "64", "--num_samples", "16", "--train_batchsize", "4", "--max_steps", "6",
                "--max_epochs", "-1", "--learning_rate", "1e-3", "--adam_beta2", "0.95", "--warmup_steps", "2",
                "--strategy", "deepspeed_stage_2", "--default_root_dir", str(tmp_path),
                "--save_ckpt_path", str(tmp_path / "ckpt"), "--load_ckpt_path", str(tmp_path / "ckpt" / "last.ckpt"),
                "--every_n_train_steps", "3", "--save_last", "--log_every_n_steps", "1", "--dataloader_workers", "0",
                *extra]
    trainer, module = ex.main(args())
    assert trainer.global_step == 6
    assert any(b["input_ids"].shape[0] < 4 for b in seen)          # samples shared rows
    assert all("segment_ids" in b for b in seen)
    import json
    losses = [json.loads(l)["train/loss"] for l in open(os.path.join(trainer.logger.save_dir, "metrics.jsonl"))]
    assert all(math.isfinite(x) for x in losses)
    ck = tmp_path / "ckpt" / "last.ckpt" / "checkpoint"
    assert (ck / "mp_rank_00_model_states.pt").exists()
    state = torch.load(ck / "mp_rank_00_model_states.pt", map_location="cpu", weights_only=False)
    assert state["global_samples"] == 6 * 4        # consumed samples: the sampler's count, not the packed rows
    w_before = module.model.flat.params.clone()
    trainer2, module2 = ex.main(args(("--max_steps", "8")))
    assert trainer2.global_step == 8
    assert getattr(module2, "consumed_samples", None) == 24
    assert not torch.equal(module2.model.flat.params, w_before)
