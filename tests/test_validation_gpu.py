"""GPU: the forward-only path that validation runs. (1) For every model class, the no-grad forward gives the same loss and logits
bits as the grad-mode forward, keeps nothing for backward, leaves the gradient buffers alone and peaks lower in memory. (2) A
validation run inside `Trainer.fit` leaves training bit-for-bit unchanged: examples/pretrain_ziya_llama.py at the small LLaMA
golden config, ZeRO-2 and ZeRO-1, GA 2, validation every 3 micro-batches (inside accumulation windows) and 2 sanity batches.
(3) Each logged val_loss is the batch-size-weighted mean of no-grad losses on that step's weights, and at the golden weights it
is within the oracle tolerance of the reference's loss."""
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "fengshen-lm_b200", "compat"), os.path.join(ROOT, "examples")):
    if p not in sys.path:
        sys.path.insert(0, p)
import hf_oracle as H  # noqa: E402  (checker only)
import llama_oracle as O  # noqa: E402  (checker only)

LLAMA_GOLD = os.path.join(ROOT, "tests", "golden", "llama_h256_hn64.npz")


def _llama():
    from fsb200.models.llama import LlamaForCausalLM
    g = np.load(LLAMA_GOLD)
    V, h, L, nh, B, S = (int(x) for x in g["config"])
    m = LlamaForCausalLM(SimpleNamespace(vocab_size=V, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                                         rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                                         llama_mlp_multiple_of=256), device="cuda")
    m.load_reference_state_dict(O.make_weights(V, h, L, seed=int(g["weight_seed"])))
    return m, O.make_batch(V, B, S, seed=int(g["batch_seed"]))


def _gpt2():
    from fsb200.models.gpt2 import GPT2LMHeadModel
    ref = H.build_gpt2(H.GPT2_SMALL)
    m = GPT2LMHeadModel(ref.config, device="cuda")
    m.load_reference_state_dict(ref.state_dict())
    b = H.make_lm_batch(H.GPT2_SMALL["vocab_size"], 2, 96, seed=1234)
    return m, {"input_ids": b["input_ids"], "labels": b["labels"]}


def _bert():
    from fsb200.models.bert import BertForMaskedLM
    ref = H.build_bert(H.BERT_SMALL)
    m = BertForMaskedLM(ref.config, device="cuda")
    m.load_reference_state_dict(ref.state_dict())
    return m, H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 3, 96, seed=5, pad_tail=20)


def _megatron_bert():
    from fsb200.models.bert import MegatronBertForPreTraining
    ref = H.build_megatron_bert(H.BERT_SMALL)
    m = MegatronBertForPreTraining(ref.config, device="cuda")
    m.load_reference_state_dict(ref.state_dict())
    return m, H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 3, 96, seed=6, nsp=True, pad_tail=11)


def _mt5():
    from fsb200.models.t5 import MT5ForConditionalGeneration
    ref = H.build_mt5(H.MT5_SMALL)
    m = MT5ForConditionalGeneration(ref.config, device="cuda")
    m.load_reference_state_dict(ref.state_dict())
    return m, H.make_t5_batch(H.MT5_SMALL["vocab_size"], 2, 96, 48, seed=7, pad_tail=13)


MODELS = {"llama": _llama, "gpt2": _gpt2, "bert": _bert, "megatron_bert_nsp": _megatron_bert, "mt5": _mt5}


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("name", sorted(MODELS))
def test_no_grad_forward_equals_grad_forward(name):
    model, batch = MODELS[name]()
    batch = {k: v.cuda() for k, v in batch.items()}
    model.flat.grads.fill_(3.0)                                  # a pattern no kernel writes
    grads_before = model.flat.grads.clone()

    def nograd():
        with torch.no_grad():
            return model(**batch, return_logits=True)
    out_n, peak_n = _peak(nograd)
    assert out_n.loss.grad_fn is None and not out_n.loss.requires_grad                 # nothing kept for backward
    assert torch.equal(model.flat.grads, grads_before)                                # gradient buffers untouched
    out_g, peak_g = _peak(lambda: model(**batch, return_logits=True))
    assert out_g.loss.grad_fn is not None
    assert torch.equal(out_n.loss, out_g.loss.detach()), (out_n.loss.item(), out_g.loss.item())
    assert torch.equal(out_n.logits, out_g.logits)
    assert peak_n < peak_g, (peak_n, peak_g)
    del out_g


# ---- the example script with validation: training is unchanged ---------------------------------------------------------------
def _val_example(set_attr, ex, snapshots):
    """examples/pretrain_ziya_llama.py with the validation of finetune_ziya_llama.py:150-153 (the forward's loss, logged with
    sync_dist) and a validation split. `set_attr(obj, name, value)` installs both classes."""

    class Llama(ex.Llama):
        def validation_step(self, batch, batch_idx):
            if batch_idx == 0 and not self.trainer.sanity_checking:
                snapshots[self.trainer.global_step] = self.model.flat.params.clone()
            loss = self(**batch).loss
            self.log('val_loss', loss, sync_dist=True)
            return loss

    class Data(ex.UniversalDataModule):
        def __init__(self, tokenizer, args, collate_fn, datasets):
            datasets = dict(datasets, validation=ex.SyntheticTokens(args.vocab_size, args.max_seq_length, 10, seed=99))
            super().__init__(tokenizer=tokenizer, args=args, collate_fn=collate_fn, datasets=datasets)

    set_attr(ex, "Llama", Llama)
    set_attr(ex, "UniversalDataModule", Data)


def _args(tmp, strategy):
    # the small LLaMA golden config (tests/golden/llama_h256_hn64.npz: V 512, h 256, 2 layers, 4 heads, seq 64)
    return ["--hidden_size", "256", "--num_layers", "2", "--num_heads", "4", "--vocab_size", "512", "--max_seq_length", "64",
            "--num_samples", "48", "--train_batchsize", "4", "--val_batchsize", "4", "--max_steps", "6", "--max_epochs", "-1",
            "--accumulate_grad_batches", "2", "--learning_rate", "1e-3", "--adam_beta2", "0.95", "--warmup_steps", "2",
            "--strategy", strategy, "--default_root_dir", str(tmp), "--save_ckpt_path", str(tmp / "ckpt"),
            "--log_every_n_steps", "1", "--dataloader_workers", "0", "--val_check_interval", "3",
            "--num_sanity_val_steps", "2"]


def _lines(trainer):
    return [json.loads(l) for l in open(os.path.join(trainer.logger.save_dir, "metrics.jsonl"))]


@pytest.mark.parametrize("strategy", ["deepspeed_stage_2", "deepspeed_stage_1"])
def test_validation_leaves_training_bit_identical(tmp_path, monkeypatch, strategy):
    import pretrain_ziya_llama as ex
    plain, _ = ex.main(_args(tmp_path / "plain", strategy))
    snapshots = {}
    with monkeypatch.context() as mp:
        _val_example(mp.setattr, ex, snapshots)
        trainer, module = ex.main(_args(tmp_path / "val", strategy))
    assert trainer.global_step == plain.global_step == 6
    assert torch.equal(trainer.engine.flat.params, plain.engine.flat.params)
    for k in ("master", "exp_avg", "exp_avg_sq"):
        assert torch.equal(getattr(trainer.engine, k), getattr(plain.engine, k)), k
    train = [l["train/loss"] for l in _lines(trainer) if "train/loss" in l]
    assert train == [l["train/loss"] for l in _lines(plain) if "train/loss" in l] and len(train) == 6
    assert not any(k.startswith("val") for l in _lines(trainer) if "train/loss" in l for k in l)
    # 12 micro-batches, a run after micro-batches 3, 6, 9, 12: global steps 1 and 4 are inside an accumulation window
    val = [(l["step"], l["val_loss"]) for l in _lines(trainer) if "val_loss" in l]
    assert [s for s, _ in val] == [1, 3, 4, 6] and sorted(snapshots) == [1, 3, 4, 6]
    # each logged value is the batch-size-weighted mean of the no-grad losses on that step's weights
    model = module.model
    loader = trainer.datamodule.val_dataloader()
    for step, logged in val:
        model.flat.params.copy_(snapshots[step])
        num, den = 0.0, 0
        with torch.no_grad():
            for b in loader:
                bs = b["input_ids"].shape[0]
                num += float(model(**{k: v.cuda() for k, v in b.items()}).loss.double()) * bs
                den += bs
        assert logged == num / den, (step, logged, num / den)


def test_logged_val_loss_at_the_golden_weights(tmp_path):
    """lr 0: after the first step the weights are still the golden ones; the logged val_loss over the golden batch is within
    the oracle tolerance of the unmodified reference's loss."""
    import pytorch_lightning as pl
    g = np.load(LLAMA_GOLD)
    batch = O.make_batch(*(int(x) for x in (g["config"][0], g["config"][4], g["config"][5])), seed=int(g["batch_seed"]))
    rows = [{k: v[i] for k, v in batch.items()} for i in range(batch["input_ids"].shape[0])]
    loader = torch.utils.data.DataLoader(rows, batch_size=len(rows))

    class Golden(pl.LightningModule):
        def setup(self, stage=None):
            self.model, _ = _llama()

        def configure_optimizers(self):
            return torch.optim.AdamW(self.parameters(), lr=0.0, weight_decay=0.0)

        def training_step(self, b, batch_idx):
            return self.model(**b).loss

        def validation_step(self, b, batch_idx):
            self.log("val_loss", self.model(**b).loss, sync_dist=True)

    trainer = pl.Trainer(strategy="deepspeed_stage_2", max_steps=1, max_epochs=None, num_sanity_val_steps=0,
                         val_check_interval=1, default_root_dir=str(tmp_path))
    trainer.fit(Golden(), train_dataloaders=loader, val_dataloaders=loader)
    got = trainer.callback_metrics["val_loss"]
    assert abs(got - float(g["loss"])) <= 3e-3, (got, float(g["loss"]))


# ---- two GPUs: data parallelism 2 and tensor parallelism 2 ---------------------------------------------------------------------
def _tp_example_module(ex):
    """The example's module with its model built under tensor parallelism (the example's own setup() insists on TP 1)."""

    class Llama(ex.Llama):
        def setup(self, stage) -> None:
            config = ex.LlamaConfig(vocab_size=self.hparams.vocab_size, hidden_size=self.hparams.hidden_size,
                                    num_hidden_layers=self.hparams.num_layers, num_attention_heads=self.hparams.num_heads)
            self.model = ex.LlamaForCausalLM(config).cuda()
            assert self.model.tp == 2
            if stage == 'fit':
                self.total_steps = ex.get_total_steps(self.trainer, self.hparams)
    return Llama


def _two_gpu_rank(rank, world, port, workdir, mode, q):
    """One rank of the ZeRO-2 / GA 2 example run, without and then with validation, on NCCL."""
    import pathlib
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import pretrain_ziya_llama as ex
    extra = []
    if mode == "tp":   # the tensor-parallel pair forms one data-parallel rank: the training sampler shards over mpu's groups
        ex.Llama = _tp_example_module(ex)
        extra = ["--model_parallel_size", "2", "--replace_sampler_ddp", "False", "--use_mpu"]
    work = pathlib.Path(workdir)
    plain, _ = ex.main(_args(work / "plain", "deepspeed_stage_2") + extra)
    snapshots = {}
    _val_example(setattr, ex, snapshots)
    trainer, _ = ex.main(_args(work / "val", "deepspeed_stage_2") + extra)
    torch.cuda.synchronize()
    same = {k: torch.equal(getattr(trainer.engine, k), getattr(plain.engine, k)) for k in ("master", "exp_avg", "exp_avg_sq")}
    same["params"] = torch.equal(trainer.engine.flat.params, plain.engine.flat.params)
    logged = None
    if rank == 0:      # rank 0 writes the logger
        a, b = _lines(plain), _lines(trainer)
        logged = ([l["train/loss"] for l in a if "train/loss" in l], [l["train/loss"] for l in b if "train/loss" in l],
                  [l["step"] for l in b if "val_loss" in l],
                  any(k.startswith("val") for l in b if "train/loss" in l for k in l))
    q.put((rank, same, logged, float(trainer.callback_metrics["val_loss"]), sorted(snapshots)))
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("mode", ["dp", "tp"])
def test_validation_leaves_training_bit_identical_on_two_gpus(tmp_path, mode):
    """DP 2: validation right after engine.step(), while the parameter all-gathers are in flight on the side stream, and in the
    middle of accumulation windows with ZeRO-2 reduce-scatters pending; the fp64 metric all-reduce on NCCL. TP 2: the no-grad
    forward's tensor-parallel all-reduces, fed one batch per tensor-parallel pair by the data-parallel validation sampler."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29931 if mode == "dp" else 29937
    procs = [ctx.Process(target=_two_gpu_rank, args=(r, 2, port, str(tmp_path), mode, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        r = q.get(timeout=600)
        res[r[0]] = r
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank in (0, 1):
        assert all(res[rank][1].values()), (rank, res[rank][1])
        assert res[rank][4] == [1, 3, 4, 6]
    train_plain, train_val, val_steps, val_in_train_lines = res[0][2]
    assert train_val == train_plain and len(train_val) == 6
    assert val_steps == [1, 3, 4, 6] and not val_in_train_lines
    assert res[0][3] == res[1][3]                                   # sync_dist: one value on every rank


def _tp_nograd_rank(rank, world, port, q):
    from fengshen.utils.llama_convert import split_state_dict_tp
    from fsb200.models.llama import LlamaForCausalLM
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    tp_group = dist.new_group(list(range(world)))
    g = np.load(LLAMA_GOLD)
    V, h, L, nh, B, S = (int(x) for x in g["config"])
    model = LlamaForCausalLM(SimpleNamespace(vocab_size=V, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                                             rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                                             llama_mlp_multiple_of=256), device=dev, world_size=1, tp_group=tp_group)
    model.load_reference_state_dict(split_state_dict_tp(O.make_weights(V, h, L, seed=int(g["weight_seed"])), world, nh)[rank])
    batch = {k: v.to(dev) for k, v in O.make_batch(V, B, S, seed=int(g["batch_seed"])).items()}
    with torch.no_grad():
        model(**batch)                                       # warm-up: NCCL communicators, rope tables
    model.flat.grads.fill_(3.0)
    before = model.flat.grads.clone()

    def nograd():
        with torch.no_grad():
            return model(**batch, return_logits=True)
    out_n, peak_n = _peak(nograd)
    untouched = torch.equal(model.flat.grads, before)
    out_g, peak_g = _peak(lambda: model(**batch, return_logits=True))
    checks = {"no_graph": out_n.loss.grad_fn is None and not out_n.loss.requires_grad, "grads_untouched": untouched,
              "graph": out_g.loss.grad_fn is not None, "loss_equal": torch.equal(out_n.loss, out_g.loss.detach()),
              "logits_equal": torch.equal(out_n.logits, out_g.logits), "lower_peak": peak_n < peak_g}
    q.put((rank, checks, float(out_n.loss), float(g["loss"])))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tensor_parallel_no_grad_forward_equals_grad_forward():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_nograd_rank, args=(r, 2, 29941, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r[0], r[1:]) for r in (q.get(timeout=300) for _ in range(2)))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank in (0, 1):
        assert all(res[rank][0].values()), (rank, res[rank][0])
    assert res[0][1] == res[1][1]                                    # gathered logits: the same loss on both ranks
    assert abs(res[0][1] - res[0][2]) <= 3e-3, (res[0][1], res[0][2])
