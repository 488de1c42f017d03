"""GPU: activation recompute for Ziya-LLaMA (LlamaForCausalLM gradient_checkpointing).

Bit-identical (torch.equal) with recompute on and off: the loss, the whole flat gradient buffer after the first micro-batch
and the parameters after 3 optimizer steps, on the three goldens, under ZeRO-1 and ZeRO-2 with gradient accumulation 2, with
fp8=True, on packed batches (segment_ids), at Ziya width with 2 layers and seq 2048, and under tensor parallelism 2 (2
GPUs); the CUDA-graph step with recompute equals the eager step with and without it. Memory: at Ziya width, seq 2048, going
from 2 to 4 layers grows the activation peak by two residual-stream checkpoints with recompute, and by at least two saved
sets without. Every launch of a recomputed Ziya-width step is checked against fp64 and for its write footprint. The API
(HF's gradient-checkpointing names, the compat from_pretrained keyword, the refusal of the other models and of a mode
change after a graph capture), unchanged no-grad and generate outputs, and the example script's --gradient_checkpointing."""
import gc
import glob
import json
import math
import os
import sys
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))
import bench  # noqa: E402  (read only: workload, build_model, make_host_batches)
import llama_oracle as O  # noqa: E402  (weights and batches of the goldens)

import footprint as F  # noqa: E402
import launch_refs as R  # noqa: E402
import test_path_launches_gpu as PL  # noqa: E402
from launch_census import Recorder, free_gib  # noqa: E402
from fsb200.engine import ZeroEngine  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402
from fsb200.packing import pack_causal_lm_batch  # noqa: E402
from fsb200.trainer import PretrainStep  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "llama_*.npz")))
EOS = 2
MIB = 2 ** 20


def _cfg(V, h, L, nh):
    return SimpleNamespace(vocab_size=V, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                           rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                           llama_mlp_multiple_of=256)


def _golden(path, **kw):
    """-> (build(), V, S): a builder of the golden's model with the reference weights loaded."""
    g = np.load(path)
    V, h, L, nh, _, S = (int(x) for x in g["config"])
    sd = O.make_weights(V, h, L, seed=int(g["weight_seed"]))

    def build():
        m = LlamaForCausalLM(_cfg(V, h, L, nh), device="cuda", **kw)
        m.load_reference_state_dict(sd)
        return m
    return build, V, S


def _ziya(layers, seq=2048, micro=1):
    w = dict(bench.workload("ziya-llama-13b"), num_hidden_layers=layers, seq=seq, micro=micro, per_gpu=micro)
    return w, (lambda: bench.build_model(w, torch.device("cuda", torch.cuda.current_device()), 1))


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _need(gib, what):
    _free()
    if free_gib() < gib:
        pytest.skip(f"{what} needs about {gib} GiB free; {free_gib():.1f} GiB are")


def _train(build, batches, recompute, stage=2, ga=1, steps=3):
    """`steps` optimizer steps of `ga` micro-batches each (batches[step][micro], dicts of device tensors) through ZeroEngine
    -> (every micro-batch's loss, the flat gradient buffer after the first micro-batch, the parameters at the end)."""
    model = build()
    if recompute:
        model.gradient_checkpointing_enable()
    eng = ZeroEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=ga, stage=stage)
    losses, g0 = [], None
    for st in range(steps):
        for mb in batches[st]:
            out = model(**mb)
            out.loss.backward()
            if g0 is None:
                g0 = model.flat.grads.clone()
            eng.backward_done()
            losses.append(out.loss.detach())
        eng.step()
    eng.wait_params()
    torch.cuda.synchronize()
    res = torch.stack(losses), g0, model.flat.params.clone()
    del model, eng
    _free()
    return res


def _assert_same(a, b):
    (la, ga, pa), (lb, gb, pb) = a, b
    assert torch.equal(la, lb), (la.tolist(), lb.tolist())
    assert torch.equal(ga, gb), "flat gradient buffer after the first micro-batch differs"
    assert torch.equal(pa, pb), "parameters after the optimizer steps differ"


def _lm_batches(V, S, steps, ga, B=2, seed=0):
    out = []
    for st in range(steps):
        mbs = []
        for m in range(ga):
            b = O.make_batch(V, B, S, seed=seed + 10 * st + m)
            mbs.append({k: b[k].cuda() for k in ("input_ids", "labels", "position_ids")})
        out.append(mbs)
    return out


def _sft_packed(V, S, n, seed):
    """Ziya-SFT-format samples (prompt unlabelled, then the labelled output) packed into rows of S with segment_ids."""
    rng = np.random.default_rng(seed)
    ids, labs = [], []
    for _ in range(n):
        p = rng.integers(3, V, int(rng.integers(1, S // 4 + 1))).tolist()
        o = rng.integers(3, V, int(rng.integers(1, S // 3 + 1))).tolist() + [EOS]
        ids.append(p + o)
        labs.append([-100] * len(p) + o)
    L = max(len(i) for i in ids)
    padded = {"input_ids": torch.tensor([i + [EOS] * (L - len(i)) for i in ids]),
              "labels": torch.tensor([l + [-100] * (L - len(l)) for l in labs]),
              "position_ids": torch.arange(L)[None].expand(n, L).contiguous()}
    return pack_causal_lm_batch(padded, S, EOS)


# ------------------------------------------------------------------------------------------------- bit-identical training
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_goldens_train_bit_identically_with_recompute(path):
    build, V, S = _golden(path)
    batches = _lm_batches(V, S, 3, 1)
    _assert_same(_train(build, batches, False), _train(build, batches, True))


@pytest.mark.parametrize("stage", [1, 2])
def test_zero_with_gradient_accumulation_is_bit_identical(stage):
    build, V, S = _golden(GOLDEN[0])
    batches = _lm_batches(V, S, 3, 2, seed=100)
    _assert_same(_train(build, batches, False, stage=stage, ga=2), _train(build, batches, True, stage=stage, ga=2))


def test_fp8_is_bit_identical():
    """fp8=True: the recompute quantises w2's input for its weight gradient without running the w2 GEMM."""
    build, V, S = _golden(GOLDEN[1], fp8=True)
    batches = _lm_batches(V, S, 3, 1, seed=200)
    _assert_same(_train(build, batches, False), _train(build, batches, True))


def test_packed_batches_are_bit_identical():
    build, V, S = _golden(GOLDEN[0])
    batches = [[{k: v.cuda() for k, v in _sft_packed(V, S, 7, seed=300 + st).items()}] for st in range(3)]
    assert all("segment_ids" in b[0] for b in batches)
    _assert_same(_train(build, batches, False), _train(build, batches, True))


def test_ziya_width_two_layers_seq_2048_is_bit_identical():
    _need(40, "two Ziya-width 2-layer models with ZeRO state, one at a time")
    w, build = _ziya(2)
    batches = [[{k: v.cuda() for k, v in b.items()} for b in bench.make_host_batches(w, 1, st)] for st in range(3)]
    off = _train(build, batches, False)
    _assert_same(off, _train(build, batches, True))


@pytest.mark.parametrize("stage", [1, 2])
def test_cuda_graph_step_with_recompute_equals_eager_with_and_without(stage):
    build, V, S = _golden(GOLDEN[0])
    batches = _lm_batches(V, S, 4, 2, seed=400)
    runs = []
    for graph, recompute in ((True, True), (False, True), (False, False)):
        model = build()
        if recompute:
            model.gradient_checkpointing_enable()
        st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, ga_steps=2,
                          stage=stage, cuda_graph=graph)
        losses = torch.stack([st.step_device(mbs) for mbs in batches])
        st.engine.wait_params()
        torch.cuda.synchronize()
        runs.append((losses, model.flat.grads.clone(), model.flat.params.clone()))
        del model, st
        _free()
    _assert_same(runs[0], runs[1])
    _assert_same(runs[1], runs[2])


# ---------------------------------------------------------------------------------------------------- tensor parallelism
TP_V, TP_H, TP_NL, TP_NH, TP_S = 512, 256, 2, 4, 128


def _tp_run(rank, port, q):
    import torch.distributed as dist
    from fengshen.utils.llama_convert import split_state_dict_tp
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=dev)
    tp_group = dist.new_group([0, 1])
    dp_group = [dist.new_group([r]) for r in range(2)][rank]
    shard = split_state_dict_tp(O.make_weights(TP_V, TP_H, TP_NL, seed=0), 2, TP_NH)[rank]
    res = []
    for recompute in (False, True):
        model = LlamaForCausalLM(_cfg(TP_V, TP_H, TP_NL, TP_NH), device=dev, world_size=1, tp_group=tp_group,
                                 gradient_checkpointing=recompute)
        model.load_reference_state_dict(shard)
        eng = ZeroEngine(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1, grad_clip=1.0, process_group=dp_group,
                         tp_group=tp_group)
        losses, g0 = [], None
        for it in range(3):
            b = O.make_batch(TP_V, 2, TP_S, seed=70 + it)
            out = model(**{k: b[k].to(dev) for k in ("input_ids", "labels", "position_ids")})
            out.loss.backward()
            if g0 is None:
                g0 = model.flat.grads.clone()
            eng.backward_done()
            eng.step()
            losses.append(out.loss.detach())
        eng.wait_params()
        res.append((torch.stack(losses), g0, model.flat.params.clone()))
    same = all(torch.equal(a, b) for a, b in zip(res[0], res[1]))
    q.put((rank, same))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tensor_parallel_2_is_bit_identical():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_run, args=(r, 29871, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(same for _, same in res), res


# -------------------------------------------------------------------------------------------------------------- memory
def _activation_peak(layers, recompute):
    """At Ziya width, seq 2048, micro-batch 1: max_memory_allocated over a forward + backward minus memory_allocated just
    before it, after a warm-up step; and the bytes of one layer's saved tuple (distinct storages), from a layer run with
    save=True."""
    w, build = _ziya(layers)
    model = build()
    if recompute:
        model.gradient_checkpointing_enable()
    b = {k: v.cuda() for k, v in bench.make_host_batches(w, 1, 0)[0].items()}

    def step():
        out = model(**b)
        out.loss.backward()
    step()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - m0
    with torch.no_grad():
        S = w["seq"]
        x = torch.randn((S, w["hidden_size"]), device="cuda").to(torch.bfloat16)
        pos = torch.arange(S, device="cuda")
        saved = model._layer(0, model._proj[0], x, None, pos, 1, S, model._attend(None), save=True)[3]
        leaves = [t for item in saved for t in (item if isinstance(item, tuple) else (item,)) if t is not None]
        tuple_bytes = sum({t.untyped_storage().data_ptr(): t.untyped_storage().nbytes() for t in leaves}.values())
    del model, b, saved, leaves, x
    _free()
    return peak, tuple_bytes


def test_activation_peak_grows_by_the_checkpoints_only():
    _need(16, "a Ziya-width 4-layer model with gradients and its activations at seq 2048")
    T, h = 2048, 5120
    on2, _ = _activation_peak(2, True)
    on4, _ = _activation_peak(4, True)
    off2, tup = _activation_peak(2, False)
    off4, _ = _activation_peak(4, False)
    print(f"\n[recompute] activation peak, 2 -> 4 layers: with {on2 / MIB:.0f} -> {on4 / MIB:.0f} MiB, without "
          f"{off2 / MIB:.0f} -> {off4 / MIB:.0f} MiB; one layer's saved tuple {tup / MIB:.0f} MiB")
    assert on4 - on2 <= 2 * T * h * 2 + 64 * MIB, (on2, on4)
    assert off4 - off2 >= 2 * tup, (off2, off4, tup)


# -------------------------------------------------------------------------------------------------- launch census
@pytest.mark.parametrize("check", ["fp64", "footprint"])
def test_every_launch_of_a_recomputed_ziya_step(check, monkeypatch):
    """The benchmark's Ziya step (seq 1024, micro-batch 1, ZeRO-2, GA 2) at 2 layers with recompute, through the census
    recorder: every launch signature against fp64 (tests/launch_refs.py), or for its write footprint (tests/footprint.py).
    The recompute adds no op, so every launch has a checker; rmsnorm_fwd runs 4 times per layer and micro-batch."""
    _need(30 if check == "fp64" else 42, f"the {check} census of a Ziya-width 2-layer step")
    t0 = time.time()
    torch.manual_seed(0)
    w = PL._two_layers(bench.workload("ziya-llama-13b"))
    model = bench.build_model(w, torch.device("cuda", torch.cuda.current_device()), 1)
    model.gradient_checkpointing_enable()
    stats = F.Stats()
    rec = Recorder(R.CHECKERS if check == "fp64" else F.footprint_checkers(stats))
    (loss, growth), ga = PL._train_step(w, model, rec, monkeypatch)
    PL._finish(f"recompute-{check}", rec, growth, t0)
    assert math.isfinite(float(loss.item()))
    n_norm = sum(n for (op, _), n in rec.calls.items() if op == "rmsnorm_fwd")
    assert n_norm == ga * (4 * model.nl + 1), n_norm
    if check == "footprint":
        assert stats.checked
    del model, loss
    _free()


# ------------------------------------------------------------------------------------------------------------------ API
def test_gradient_checkpointing_switches():
    build, V, S = _golden(GOLDEN[0])
    m = build()
    assert LlamaForCausalLM.supports_gradient_checkpointing
    assert not m.is_gradient_checkpointing
    m.gradient_checkpointing_enable()
    assert m.is_gradient_checkpointing
    m.gradient_checkpointing_disable()
    assert not m.is_gradient_checkpointing
    m.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    assert m.is_gradient_checkpointing
    g = np.load(GOLDEN[0])
    V, h, L, nh, _, S = (int(x) for x in g["config"])
    assert LlamaForCausalLM(_cfg(V, h, L, nh), device="cuda", gradient_checkpointing=True).is_gradient_checkpointing


def test_compat_from_pretrained_passes_the_flag(tmp_path):
    from fengshen.models.llama.configuration_llama import LlamaConfig
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    cfg = LlamaConfig(vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, rms_norm_epsilon=1e-6)
    Compat(cfg, device="cuda", seed=7).save_pretrained(str(tmp_path))
    assert Compat.from_pretrained(str(tmp_path), gradient_checkpointing=True).is_gradient_checkpointing
    assert not Compat.from_pretrained(str(tmp_path)).is_gradient_checkpointing


@pytest.mark.parametrize("family", ["gpt2", "bert", "megatron", "t5"])
def test_other_models_refuse_gradient_checkpointing(family):
    w = {"gpt2": dict(family="gpt2", vocab_size=512, n_positions=128, n_embd=128, n_layer=1, n_head=2),
         "bert": dict(family="bert", variant="bert", vocab_size=512, hidden_size=128, num_hidden_layers=1,
                      num_attention_heads=2, intermediate_size=256, hidden_act="gelu"),
         "megatron": dict(family="bert", variant="megatron", vocab_size=512, hidden_size=128, num_hidden_layers=1,
                          num_attention_heads=2, intermediate_size=256, hidden_act="gelu"),
         "t5": dict(family="t5", vocab_size=512, d_model=128, d_kv=64, d_ff=256, num_layers=1, num_heads=2)}[family]
    m = bench.build_model(w, torch.device("cuda", torch.cuda.current_device()), 1)
    assert not m.supports_gradient_checkpointing and not m.is_gradient_checkpointing
    with pytest.raises(NotImplementedError, match=type(m).__name__):
        m.gradient_checkpointing_enable()
    assert not m.is_gradient_checkpointing
    m.gradient_checkpointing_disable()


def test_mode_change_after_graph_capture_raises():
    build, V, S = _golden(GOLDEN[0])
    model = build()
    st = PretrainStep(model, lambda s_: 1e-3, lr=1e-3, cuda_graph=True)
    batches = _lm_batches(V, S, 2, 1, seed=500)
    st.step_device(batches[0])
    model.gradient_checkpointing_enable()
    with pytest.raises(RuntimeError, match="gradient checkpointing off"):
        st.step_device(batches[1])
    model.gradient_checkpointing_disable()
    assert math.isfinite(float(st.step_device(batches[1])))


def test_no_grad_forward_and_generate_are_unchanged():
    build, V, S = _golden(GOLDEN[1])
    model = build()
    b = O.make_batch(V, 2, S, seed=600)
    batch = {k: b[k].cuda() for k in ("input_ids", "labels", "position_ids")}
    prompt = b["input_ids"][:, :16].cuda()
    outs = []
    for recompute in (False, True):
        if recompute:
            model.gradient_checkpointing_enable()
        with torch.no_grad():
            o = model(**batch, return_logits=True)
        outs.append((o.loss, o.logits, model.generate(prompt, max_new_tokens=8, pad_token_id=0)))
    (l0, g0, t0), (l1, g1, t1) = outs
    assert torch.equal(l0, l1) and torch.equal(g0, g1) and torch.equal(t0, t1)


# -------------------------------------------------------------------------------------------------------------- example
def test_example_script_with_gradient_checkpointing_trains_checkpoints_and_resumes(tmp_path):
    """examples/pretrain_ziya_llama.py --gradient_checkpointing trains 6 steps, checkpoints and resumes to 8; every logged
    loss and the final parameters equal those of the same runs without the flag."""
    if os.path.join(ROOT, "examples") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "examples"))
    import pretrain_ziya_llama as ex

    def args(d, extra=()):
        return ["--hidden_size", "256", "--num_layers", "2", "--num_heads", "4", "--vocab_size", "512",
                "--max_seq_length", "64", "--num_samples", "16", "--train_batchsize", "4", "--max_steps", "6",
                "--max_epochs", "-1", "--learning_rate", "1e-3", "--adam_beta2", "0.95", "--warmup_steps", "2",
                "--strategy", "deepspeed_stage_2", "--default_root_dir", str(d),
                "--save_ckpt_path", str(d / "ckpt"), "--load_ckpt_path", str(d / "ckpt" / "last.ckpt"),
                "--every_n_train_steps", "3", "--save_last", "--log_every_n_steps", "1", "--dataloader_workers", "0",
                *extra]
    runs = []
    for flag in ((), ("--gradient_checkpointing",)):
        d = tmp_path / ("on" if flag else "off")
        trainer, module = ex.main(args(d, flag))
        assert trainer.global_step == 6
        assert module.model.is_gradient_checkpointing == bool(flag)
        assert (d / "ckpt" / "last.ckpt" / "checkpoint" / "mp_rank_00_model_states.pt").exists()
        trainer2, module2 = ex.main(args(d, flag + ("--max_steps", "8")))
        assert trainer2.global_step == 8
        assert getattr(module2, "consumed_samples", None) == 24
        losses = [json.loads(l)["train/loss"] for l in open(os.path.join(trainer2.logger.save_dir, "metrics.jsonl"))
                  if "train/loss" in json.loads(l)]
        assert len(losses) >= 8 and all(math.isfinite(x) for x in losses)
        runs.append((losses, module2.model.flat.params.clone()))
        del trainer, module, trainer2, module2
        _free()
    assert runs[0][0] == runs[1][0], runs
    assert torch.equal(runs[0][1], runs[1][1])
