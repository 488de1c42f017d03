"""CPU: validation inside the compat `Trainer.fit` — PL 1.9's cadence, limits and sanity pass, the batch-size-weighted metric
aggregation (per rank and over gloo ranks), the data-parallel sharding of validation batches under tensor parallelism, and a
recipe whose module carries the reference's own `validation_step`. The model is tests/toy_models.py's GPT-2 double, the engine
kernels are tests/cpu_kernels.py (as in tests/test_hf_trainer_flow_cpu.py)."""
import json
import os
import sys
from types import SimpleNamespace

import pytest
import torch

import hf_fixtures as F

for p in (os.path.join(F.ROOT, "fengshen-lm_b200", "compat"), os.path.join(F.ROOT, "fengshen-lm_b200"),
          os.path.join(F.ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

N_TRAIN, N_VAL, BS = 12, 9, 2          # 6 training batches per epoch; 5 validation batches, the last one of 1 sample


@pytest.fixture
def cpu_engine(monkeypatch):
    import cpu_kernels
    import fsb200.engine as engine

    class CpuEngine(engine.ZeroEngine):
        def __init__(self, model, **kw):
            kw.setdefault("kernels", cpu_kernels)
            super().__init__(model, **kw)
    monkeypatch.setattr(engine, "ZeroEngine", CpuEngine)


def _rows(n, seed):
    g = torch.Generator().manual_seed(seed)
    return [{"input_ids": torch.randint(0, 32, (8,), generator=g), "value": torch.tensor(float(i))} for i in range(n)]


def _collate(rows):
    ids = torch.stack([r["input_ids"] for r in rows])
    return {"input_ids": ids, "labels": ids.clone(), "value": torch.stack([r["value"] for r in rows])}


def _loader(rows):
    return torch.utils.data.DataLoader(rows, batch_size=BS, collate_fn=_collate)


def _module_classes():
    import pytorch_lightning as pl
    import toy_models as T

    class Data(pl.LightningDataModule):
        def __init__(self, n_val=N_VAL, val_rows=None):
            super().__init__()
            self.val_calls = 0
            self.train_rows, self.val_rows = _rows(N_TRAIN, 0), val_rows or _rows(n_val, 1)

        def train_dataloader(self):
            return _loader(self.train_rows)

        def val_dataloader(self):
            self.val_calls += 1
            return _loader(self.val_rows)

    class Train(pl.LightningModule):
        """No validation_step: validation is off whatever the flags say."""

        def __init__(self):
            super().__init__()
            self.events, self.train_idx = [], None
            self.val_seen_in_training = []

        def setup(self, stage=None):
            self.model = T.ToyGPT2(SimpleNamespace(vocab_size=32, n_positions=16))

        def configure_optimizers(self):
            return torch.optim.AdamW(self.parameters(), lr=1e-2)

        def training_step(self, batch, batch_idx):
            self.train_idx = batch_idx
            self.val_seen_in_training.append(sorted(k for k in self.trainer.callback_metrics if k.startswith("val")))
            out = self.model(input_ids=batch["input_ids"], labels=batch["labels"])
            self.log("train_loss", out.loss)
            return out.loss

    class Val(Train):
        def validation_step(self, batch, batch_idx):
            assert not torch.is_grad_enabled() and not self.training
            sanity = self.trainer.sanity_checking
            self.events.append((self.current_epoch, None if sanity else self.train_idx, self.global_step, batch_idx))
            out = self.model(input_ids=batch["input_ids"], labels=batch["labels"])
            self.log("val_loss", out.loss, sync_dist=True)
            self.log("val_value", batch["value"].mean(), sync_dist=True)
            self.log("val_own", batch["value"].mean())
            return out.loss

    return pl, Data, Train, Val


def _runs(events):
    """(epoch, training batch_idx or None for the sanity pass, global_step, number of validation batches) per run."""
    runs = []
    for ep, ti, gs, vi in events:
        if vi == 0:
            runs.append([ep, ti, gs, 0])
        assert vi == runs[-1][3]
        runs[-1][3] += 1
    return [tuple(r) for r in runs]


def _fit(tmp_path, module_cls=None, data=None, ckpt=None, **kw):
    pl, Data, _, Val = _module_classes()
    kw.setdefault("num_sanity_val_steps", 0)
    kw.setdefault("max_epochs", 1)
    trainer = pl.Trainer(strategy="deepspeed_stage_2", log_every_n_steps=1, default_root_dir=str(tmp_path),
                         logger=pl.loggers.TensorBoardLogger(save_dir=str(tmp_path)), **kw)
    module = (module_cls or Val)()
    data = data or Data()
    trainer.fit(module, data, ckpt_path=ckpt)
    return trainer, module, data


# (Trainer keywords, the runs derived by hand from PL 1.9's rules; 6 training batches per epoch, 5 validation batches)
CADENCE = {
    # float: val_check_batch = int(6 * 0.5) = 3 -> after batches 2 and 5 of every epoch
    "float_half": (dict(val_check_interval=0.5, max_epochs=2), [(0, 2, 3, 5), (0, 5, 6, 5), (1, 2, 9, 5), (1, 5, 12, 5)]),
    # default 1.0: once per epoch, after its last batch
    "default": (dict(max_epochs=2), [(0, 5, 6, 5), (1, 5, 12, 5)]),
    # int within the epoch: batch 3 of every epoch, no run at the epoch's end
    "int_per_epoch": (dict(val_check_interval=4, max_epochs=2), [(0, 3, 4, 5), (1, 3, 10, 5)]),
    # int across epochs (check_val_every_n_epoch=None): total batch indices 3, 7, 11
    "int_total": (dict(val_check_interval=4, check_val_every_n_epoch=None, max_epochs=2),
                  [(0, 3, 4, 5), (1, 1, 8, 5), (1, 5, 12, 5)]),
    "every_2nd_epoch": (dict(check_val_every_n_epoch=2, max_epochs=4), [(1, 5, 12, 5), (3, 5, 24, 5)]),
    "limit_fraction": (dict(limit_val_batches=0.5), [(0, 5, 6, 2)]),                  # int(5 * 0.5)
    "limit_count": (dict(limit_val_batches=3), [(0, 5, 6, 3)]),
    "limit_zero": (dict(limit_val_batches=0, num_sanity_val_steps=2), []),
    "sanity_2": (dict(num_sanity_val_steps=2), [(0, None, 0, 2), (0, 5, 6, 5)]),
    "sanity_all": (dict(num_sanity_val_steps=-1), [(0, None, 0, 5), (0, 5, 6, 5)]),
    "sanity_all_limited": (dict(num_sanity_val_steps=-1, limit_val_batches=3), [(0, None, 0, 3), (0, 5, 6, 3)]),
    # GA 2: batches are micro-batches; the run after batch 2 falls inside the second accumulation window (global_step 1)
    "ga2": (dict(val_check_interval=3, accumulate_grad_batches=2), [(0, 2, 1, 5), (0, 5, 3, 5)]),
    # max_steps 5 stops after batch 4: runs after batches 1 and 3, none at the stop
    "max_steps": (dict(val_check_interval=2, max_steps=5, max_epochs=None), [(0, 1, 2, 5), (0, 3, 4, 5)]),
}


@pytest.mark.parametrize("case", sorted(CADENCE))
def test_cadence_table(case, tmp_path, cpu_engine):
    kw, want = CADENCE[case]
    trainer, module, data = _fit(tmp_path, **kw)
    assert _runs(module.events) == want
    assert data.val_calls == (0 if kw.get("limit_val_batches") == 0 else 1)


def test_cadence_on_resume(tmp_path, cpu_engine):
    """The sanity pass runs again on resume; the total batch index continues from global_step x GA."""
    kw = dict(val_check_interval=2, check_val_every_n_epoch=None, num_sanity_val_steps=1, max_epochs=None)
    trainer, module, _ = _fit(tmp_path / "a", max_steps=3, **kw)
    assert _runs(module.events) == [(0, None, 0, 1), (0, 1, 2, 5)]
    trainer.save_checkpoint(str(tmp_path / "ck"))
    trainer2, module2, _ = _fit(tmp_path / "b", max_steps=6, ckpt=str(tmp_path / "ck"), **kw)
    # resumed at global_step 3 (total batch index 3): the loader restarts at batch 0 = total index 3
    assert _runs(module2.events) == [(0, None, 3, 1), (0, 0, 4, 5), (0, 2, 6, 5)]
    assert trainer2.global_step == 6


def test_int_interval_longer_than_the_epoch_is_an_error(tmp_path, cpu_engine):
    with pytest.raises(ValueError, match="val_check_interval"):
        _fit(tmp_path, val_check_interval=7)
    trainer, module, _ = _fit(tmp_path / "b", val_check_interval=7, check_val_every_n_epoch=None, max_epochs=2)
    assert _runs(module.events) == [(1, 0, 7, 5)]                # total batch index 6 = epoch 1, batch 0


def test_float_interval_without_epoch_cadence_is_an_error(tmp_path, cpu_engine):
    with pytest.raises(ValueError, match="should be an integer"):
        _fit(tmp_path, val_check_interval=0.5, check_val_every_n_epoch=None)


def test_empty_validation_loader_means_no_validation(tmp_path, cpu_engine):
    _, Data, _, _ = _module_classes()

    class Empty(Data):
        def val_dataloader(self):
            return _loader([])
    for limit in (None, 0.5, 3):
        trainer, module, _ = _fit(tmp_path / str(limit), data=Empty(), limit_val_batches=limit, num_sanity_val_steps=2)
        assert module.events == [] and trainer.global_step == 6


def test_no_validation_step_means_no_validation(tmp_path, cpu_engine):
    _, Data, Train, _ = _module_classes()
    trainer, module, data = _fit(tmp_path, module_cls=Train, num_sanity_val_steps=2, val_check_interval=1)
    assert data.val_calls == 0 and trainer.global_step == 6 and not any(k.startswith("val") for k in trainer.callback_metrics)


def test_val_dataloader_errors_propagate(tmp_path, cpu_engine):
    _, Data, _, _ = _module_classes()

    class Broken(Data):
        def val_dataloader(self):
            raise KeyError("validation")
    with pytest.raises(KeyError, match="validation"):
        _fit(tmp_path, data=Broken())


def test_argparse_keeps_int_and_float_apart():
    import argparse
    import pytorch_lightning as pl
    p = pl.Trainer.add_argparse_args(argparse.ArgumentParser())
    a = p.parse_args(["--val_check_interval", "100", "--limit_val_batches", "0.1"])
    assert a.val_check_interval == 100 and isinstance(a.val_check_interval, int)
    assert a.limit_val_batches == 0.1 and isinstance(a.limit_val_batches, float)
    a = p.parse_args(["--val_check_interval", "0.1", "--limit_val_batches", "3"])
    assert isinstance(a.val_check_interval, float) and a.limit_val_batches == 3 and isinstance(a.limit_val_batches, int)
    assert p.parse_args([]).num_sanity_val_steps == 2                           # PL's default
    t = pl.Trainer.from_argparse_args(p.parse_args(["--val_check_interval", "1.0"]))
    assert t.val_check_interval == 1.0 and isinstance(t.val_check_interval, float)


def test_generate_no_tp_flags_turn_validation_off(tmp_path, cpu_engine):
    """ziya_llama/generate_no_tp.sh passes `--num_sanity_val_steps 0 --limit_val_batches 0`."""
    import argparse
    import pytorch_lightning as pl
    args = pl.Trainer.add_argparse_args(argparse.ArgumentParser()).parse_args(
        ["--num_sanity_val_steps", "0", "--limit_val_batches", "0", "--max_epochs", "1", "--log_every_n_steps", "1"])
    _, Data, _, Val = _module_classes()
    trainer = pl.Trainer.from_argparse_args(args, strategy="deepspeed_stage_2")
    module, data = Val(), Data()
    trainer.fit(module, data)
    assert module.events == [] and data.val_calls == 0 and trainer.global_step == 6


def _metric_lines(trainer):
    return [json.loads(l) for l in open(os.path.join(trainer.logger.save_dir, "metrics.jsonl"))]


def test_weighted_mean_sanity_discarded_and_clean_training_lines(tmp_path, cpu_engine):
    trainer, module, _ = _fit(tmp_path, num_sanity_val_steps=2, val_check_interval=0.5, max_epochs=1)
    # values 0..8 in batches of 2, 2, 2, 2, 1: the batch-size-weighted mean is 36 / 9 = 4 (the unweighted one would be 4.4)
    assert trainer.callback_metrics["val_value"] == 4.0 and trainer.callback_metrics["val_own"] == 4.0
    lines = _metric_lines(trainer)
    train_lines = [l for l in lines if "train_loss" in l]
    val_lines = [l for l in lines if "val_loss" in l]
    assert len(train_lines) == 6 and not any(k.startswith("val") for l in train_lines for k in l)
    assert [l["step"] for l in val_lines] == [3, 6] and all(l["val_value"] == 4.0 for l in val_lines)
    assert all(set(l) == {"step", "val_loss", "val_value", "val_own"} for l in val_lines)
    # the sanity pass (before batch 0) left nothing behind; the run after batch 2 is visible from batch 3 on
    assert module.val_seen_in_training[:3] == [[], [], []]
    assert module.val_seen_in_training[3] == ["val_loss", "val_own", "val_value"]
    # the logged val_loss is the weighted mean of the per-batch no-grad losses on the final weights
    sums = [0.0, 0]
    with torch.no_grad():
        for b in _loader(_rows(N_VAL, 1)):
            sums[0] += float(module.model(input_ids=b["input_ids"], labels=b["labels"]).loss.double()) * b["input_ids"].shape[0]
            sums[1] += b["input_ids"].shape[0]
    assert trainer.callback_metrics["val_loss"] == sums[0] / sums[1]


def test_validation_leaves_training_unchanged(tmp_path, cpu_engine):
    """ZeRO-2, GA 2, a run every 3 micro-batches (inside accumulation windows) and a sanity pass: same parameters, optimizer
    state and logged training losses as the run without validation."""
    _, Data, Train, Val = _module_classes()
    kw = dict(val_check_interval=3, accumulate_grad_batches=2, num_sanity_val_steps=2, max_epochs=2)
    a, ma, _ = _fit(tmp_path / "a", module_cls=Val, **kw)
    b, mb, _ = _fit(tmp_path / "b", module_cls=Train, **kw)
    assert len(ma.events) > 0 and mb.events == []
    assert torch.equal(ma.model.flat.params, mb.model.flat.params)
    for k in ("master", "exp_avg", "exp_avg_sq"):
        assert torch.equal(getattr(a.engine, k), getattr(b.engine, k)), k
    assert [l["train_loss"] for l in _metric_lines(a) if "train_loss" in l] == \
        [l["train_loss"] for l in _metric_lines(b) if "train_loss" in l]


# ---- two gloo ranks: the global weighted mean under sync_dist, each rank's own mean without it ---------------------------------
def _sync_rank(rank, world, port, workdir, q):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port), CUDA_VISIBLE_DEVICES="")
    for p in (os.path.join(F.ROOT, "fengshen-lm_b200", "compat"), os.path.join(F.ROOT, "fengshen-lm_b200"),
              os.path.join(F.ROOT, "tests")):
        sys.path.insert(0, p)
    import cpu_kernels
    import fsb200.engine as engine

    class CpuEngine(engine.ZeroEngine):
        def __init__(self, model, **kw):
            kw.setdefault("kernels", cpu_kernels)
            super().__init__(model, **kw)
    engine.ZeroEngine = CpuEngine
    pl, Data, _, Val = _module_classes()
    # rank 0: values 1, 2, 3 (batches of 2 and 1); rank 1: 10, 20, 30, 40 (batches of 2 and 2)
    vals = [1.0, 2.0, 3.0] if rank == 0 else [10.0, 20.0, 30.0, 40.0]
    rows = [{"input_ids": torch.arange(8) + i, "value": torch.tensor(v)} for i, v in enumerate(vals)]
    trainer = pl.Trainer(strategy="deepspeed_stage_2", max_epochs=1, num_sanity_val_steps=0, log_every_n_steps=1,
                         logger=pl.loggers.TensorBoardLogger(save_dir=workdir))
    module = Val()
    trainer.fit(module, Data(), val_dataloaders=_loader(rows))
    q.put((rank, float(trainer.callback_metrics["val_value"]), float(trainer.callback_metrics["val_own"])))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def _spawn(target, world, port, *args, timeout=240):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world, port, *args, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = {}
        for _ in range(world):
            item = q.get(timeout=timeout)
            got[item[0]] = item[1:]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
    assert all(p.exitcode == 0 for p in procs)
    return got


def test_sync_dist_over_two_gloo_ranks(tmp_path):
    got = _spawn(_sync_rank, 2, 29681, str(tmp_path))
    glob = (1 + 2 + 3 + 10 + 20 + 30 + 40) / 7
    assert got[0][0] == got[1][0] == glob
    assert got[0][1] == 2.0 and got[1][1] == 25.0
    lines = [json.loads(l) for l in open(tmp_path / "default" / "metrics.jsonl")]
    assert [l["val_value"] for l in lines if "val_value" in l] == [glob]                    # rank 0 writes once


# ---- TP 2 x DP 2 over gloo: one batch per tensor-parallel group, disjoint shards across data-parallel ranks ----------------------
def _tp_rank(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    for p in (os.path.join(F.ROOT, "fengshen-lm_b200", "compat"), os.path.join(F.ROOT, "fengshen-lm_b200")):
        sys.path.insert(0, p)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from fengshen.data.universal_datamodule import UniversalDataModule
    from fengshen.models.megatron import mpu
    mpu.initialize_model_parallel(2)
    import argparse
    args = argparse.Namespace(val_batchsize=2, val_datasets_field="validation", dataloader_workers=0)
    dm = UniversalDataModule(tokenizer=None, collate_fn=lambda xs: torch.tensor(xs), args=args,
                             datasets={"validation": list(range(12))})
    dm.trainer = SimpleNamespace(world_size=world, global_rank=rank)
    q.put((rank, [b.tolist() for b in dm.val_dataloader()]))
    dist.barrier()
    dist.destroy_process_group()


def test_validation_batches_follow_the_data_parallel_group():
    got = _spawn(_tp_rank, 4, 29683)
    idx = {r: got[r][0] for r in range(4)}
    # TP groups {0, 1} and {2, 3}; DP groups {0, 2} and {1, 3}
    assert idx[0] == idx[1] and idx[2] == idx[3]
    flat0, flat2 = sum(idx[0], []), sum(idx[2], [])
    assert not set(flat0) & set(flat2) and sorted(flat0 + flat2) == list(range(12))


# ---- recipe: the reference's validation_step bodies, run through fsb200.launch -----------------------------------------------
@pytest.fixture
def launched_t5(monkeypatch):
    saved_path = list(sys.path)
    for k in [k for k in sys.modules if k.split(".")[0] in ("fengshen", "pytorch_lightning", "deepspeed")]:
        monkeypatch.delitem(sys.modules, k)
    import cpu_kernels
    import fsb200.engine as engine
    import fsb200.hf as hf
    import fsb200.launch as launch
    import hf_recipes as R
    import toy_models as T

    class CpuEngine(engine.ZeroEngine):
        def __init__(self, model, **kw):
            kw.setdefault("kernels", cpu_kernels)
            super().__init__(model, **kw)
    monkeypatch.setattr(engine, "ZeroEngine", CpuEngine)
    monkeypatch.setattr(hf, "MT5ForConditionalGeneration",
                        type("MT5ForConditionalGeneration", (hf._HFSurface, T.ToyMT5), {"config_name": "MT5Config"}))
    monkeypatch.setattr(hf, "MegatronBertForPreTraining",
                        type("MegatronBertForPreTraining", (hf._HFSurface, T.ToyMegatronBert), {"config_name": "MegatronBertConfig"}))
    launch.prepare(R.EXAMPLE)
    hf.install()
    yield
    hf.uninstall()
    sys.path[:] = saved_path


def test_t5_recipe_validation_step_logs_val_loss_and_acc(launched_t5, tmp_path):
    """pretrain_t5.py's module with the validation of pretrain_t5.py:89-102 (loss and arg-max accuracy) restated, the
    launcher's `--val_check_interval` as a fraction of the epoch (pretrain_randeng_t5_large.sh:89)."""
    import argparse
    import pytorch_lightning as pl
    from pytorch_lightning import Trainer, loggers
    from transformers import MT5Config, MT5ForConditionalGeneration
    from fengshen.data.t5_dataloader.t5_datasets import UnsuperviseT5DataModel
    from fengshen.models.model_utils import add_module_args, configure_optimizers
    F.t5_dir(tmp_path / "m")
    F.t5_tokenised_dir(tmp_path / "tok")

    class MT5PretrainModel(pl.LightningModule):
        def __init__(self, args):
            super().__init__()
            self.save_hyperparameters(args)
            self.model = MT5ForConditionalGeneration(MT5Config.from_pretrained(args.pretrained_model_path))

        def setup(self, stage) -> None:
            self.total_steps = 12

        def configure_optimizers(self):
            return configure_optimizers(self)

        def training_step(self, batch, batch_idx):
            output = self.model(input_ids=batch['input_ids'], labels=batch['labels'])
            self.log('train_loss', output.loss, sync_dist=True)
            return output.loss

        def validation_step(self, batch, batch_idx):
            # what pretrain_t5.py:89-102 logs: the loss, and the share of all label positions (padding included) whose
            # arg-max is the label
            out = self.model(input_ids=batch['input_ids'], labels=batch['labels'])
            hits = (out.logits.argmax(-1).reshape(-1) == batch['labels'].reshape(-1).float()).float().sum()
            self.log('val_loss', out.loss, sync_dist=True)
            self.log('val_acc', hits / batch['labels'].numel(), sync_dist=True)

    p = argparse.ArgumentParser("Pretrain Unsupervise.")
    p.add_argument('--pretrained_model_path', default=None, type=str)
    p.add_argument('--new_vocab_path', default=None, type=str)
    p.add_argument('--max_seq_length', default=1024, type=int)
    p = add_module_args(p)
    p = UnsuperviseT5DataModel.add_data_specific_args(p)
    p = Trainer.add_argparse_args(p)
    args = p.parse_args(["--pretrained_model_path", str(tmp_path / "m"), "--tokenizer_type", "bert_tokenizer",
                         "--train_data_path", str(tmp_path / "tok"), "--train_split_size", "0.999", "--max_seq_length", "64",
                         "--train_batchsize", "4", "--valid_batchsize", "4", "--dataloader_num_workers", "0",
                         "--max_epochs", "1", "--learning_rate", "2e-2", "--warmup_ratio", "0.1",
                         "--strategy", "deepspeed_stage_2", "--log_every_n_steps", "1", "--default_root_dir", str(tmp_path),
                         "--val_check_interval", "0.25", "--precision", "bf16"])
    data_model = UnsuperviseT5DataModel(args)
    model = MT5PretrainModel(args)
    logger = loggers.TensorBoardLogger(save_dir=os.path.join(args.default_root_dir, 'logs/'))
    trainer = Trainer.from_argparse_args(args, logger=logger)
    trainer.fit(model, data_model)
    assert trainer.global_step == 12                               # 48 chunks / 4
    lines = _metric_lines(trainer)
    val = [l for l in lines if "val_loss" in l]
    assert [l["step"] for l in val] == [3, 6, 9, 12]               # val_check_batch = int(12 * 0.25) = 3
    assert all(set(l) == {"step", "val_loss", "val_acc"} and 0.0 <= l["val_acc"] <= 1.0 and l["val_loss"] > 0 for l in val)
    assert len([l for l in lines if "train_loss" in l]) == 12


def test_erlangshen_recipe_validation_step(launched_t5, tmp_path, monkeypatch):
    """The example's Erlangshen module with the validation of pretrain_erlangshen.py:187-190 restated (the forward's loss,
    logged with sync_dist) and a --val_file split, default cadence
    (once per epoch) plus the default 2 sanity batches."""
    import runpy
    import hf_recipes as R
    from pytorch_lightning import Trainer
    from pytorch_lightning.loggers import TensorBoardLogger
    from transformers import AutoTokenizer
    from fengshen.data.universal_datamodule import UniversalDataModule
    monkeypatch.delenv("PL_DEEPSPEED_CONFIG_PATH", raising=False)
    F.bert_dir(tmp_path / "m")
    train = F.bert_corpus(tmp_path / "train.json", n=32)
    val = F.bert_corpus(tmp_path / "val.json", n=12)
    ns = runpy.run_path(R.EXAMPLE, run_name="example_not_main")

    class ErLangShenBert(ns["ErLangShenBert"]):
        def validation_step(self, batch, batch_idx):
            loss = self(**batch).loss
            self.log('val_loss', loss, sync_dist=True)
            return loss

    args = ns["parse_args"](["--model_path", str(tmp_path / "m"), "--train_file", str(train), "--val_file", str(val),
                             "--train_batchsize", "4", "--val_batchsize", "4", "--max_seq_length", "64", "--max_epochs", "2",
                             "--learning_rate", "2e-2", "--strategy", "deepspeed_stage_1", "--replace_sampler_ddp", "False",
                             "--dataloader_workers", "0", "--log_every_n_steps", "1", "--default_root_dir", str(tmp_path),
                             "--val_check_interval", "1.0"])
    tokenizer = AutoTokenizer.from_pretrained(args.model_path)
    dm = ns["build_data"](args, tokenizer)
    dm.datasets[args.val_datasets_field] = ns["JsonLines"](args.val_file)
    module = ErLangShenBert(args, tokenizer=tokenizer)
    trainer = Trainer.from_argparse_args(args, logger=TensorBoardLogger(save_dir=str(tmp_path / "logs"), name="e"))
    trainer.fit(module, dm)
    assert trainer.global_step == 16
    val_steps = [l["step"] for l in _metric_lines(trainer) if "val_loss" in l]
    assert val_steps == [8, 16]
