"""The two HF-backed recipes as test bodies, shared by tests/test_hf_scripts_gpu.py (real fsb200 models on a GPU) and
tests/test_hf_trainer_flow_cpu.py (tests/toy_models.py doubles + tests/cpu_kernels.py): launcher -> transformers rebinding ->
script -> compat Trainer -> ZeroEngine -> checkpoints -> resume -> export. Only the loss thresholds differ between the two."""
import json
import os
import runpy

import torch

import hf_fixtures as F

EXAMPLE = os.path.join(F.ROOT, "examples", "pretrain_erlangshen_bert.py")


def losses_of(trainer):
    return [json.loads(l)["train_loss"] for l in open(os.path.join(trainer.logger.save_dir, "metrics.jsonl"))]


def erlangshen_recipe(tmp_path, monkeypatch, min_drop, lr="1e-3"):
    """examples/pretrain_erlangshen_bert.py (structure of pretrain_erlangshen.py:126-240) under the recipe's DeepSpeed JSON
    (pretrain_erlangshen_base.sh:24-39: ZeRO-1, gradient_clipping 2; bf16 instead of fp16): one epoch, then a resumed second."""
    F.bert_dir(tmp_path / "m")
    corpus = F.bert_corpus(tmp_path / "train.json", n=64)
    ds_json = tmp_path / "ds_config.json"
    ds_json.write_text(json.dumps({"zero_optimization": {"stage": 1}, "bf16": {"enabled": True}, "gradient_clipping": 2,
                                   "train_micro_batch_size_per_gpu": 4}))
    monkeypatch.setenv("PL_DEEPSPEED_CONFIG_PATH", str(ds_json))
    ns = runpy.run_path(EXAMPLE, run_name="example_not_main")
    assert ns["MegatronBertForPreTraining"].__module__ in ("fsb200.hf", "toy_models", __name__) or \
        ns["MegatronBertForPreTraining"].__name__ == "MegatronBertForPreTraining"

    def argv(epochs):
        return ["--model_path", str(tmp_path / "m"), "--train_file", str(corpus), "--train_batchsize", "4",
                "--max_seq_length", "64", "--max_epoch", str(epochs), "--learning_rate", lr, "--weight_decay", "0.1",
                "--warmup_ratio", "0.1", "--strategy", "deepspeed_stage_1", "--replace_sampler_ddp", "False",
                "--dataloader_workers", "0", "--log_every_n_steps", "1", "--default_root_dir", str(tmp_path),
                "--save_ckpt_path", str(tmp_path / "ckpt"), "--load_ckpt_path", str(tmp_path / "ckpt" / "last.ckpt"),
                "--save_last", "--every_n_train_steps", "8", "--precision", "bf16"]

    trainer, module = ns["main"](argv(1))
    assert trainer.global_step == 16 and trainer.engine.stage == 1 and trainer.engine.grad_clip == 2.0
    losses = losses_of(trainer)
    assert len(losses) == 16 and all(l == l and l < 20 for l in losses)
    assert sum(losses[-3:]) / 3 < sum(losses[:3]) / 3 - min_drop, losses
    assert 0.0 <= float(trainer.callback_metrics["train_acc"]) <= 1.0
    ck = tmp_path / "ckpt" / "last.ckpt" / "checkpoint"
    state = torch.load(ck / "mp_rank_00_model_states.pt", map_location="cpu", weights_only=False)
    assert state["global_step"] == 16 and state["global_samples"] == 64 and state["epoch"] == 1
    assert "model.bert.embeddings.word_embeddings.weight" in state["module"]
    assert (ck / "zero_pp_rank_0_mp_rank_00_optim_states.pt").exists()
    w_before = module.model.flat.params.clone()
    # second epoch resumes from last.ckpt: step counter, sample counter, LR schedule position and optimizer shard restored
    trainer2, module2 = ns["main"](argv(2))
    assert trainer2.global_step == 32
    assert module2.consumed_samples == 64 and trainer2.fit_loop.epoch_loop._batches_that_stepped == 32
    assert not torch.equal(module2.model.flat.params, w_before)
    assert trainer2.lr_scheduler_configs[0]["scheduler"].last_epoch == 32               # schedule position restored (16) + 16
    # HF-style export of the trained weights, read back under the transformers class name
    out = tmp_path / "export"
    module2.model.save_pretrained(str(out))
    again = ns["MegatronBertForPreTraining"].from_pretrained(str(out))
    sd_a, sd_b = again.state_dict(), module2.model.state_dict()
    assert sd_a.keys() == sd_b.keys()
    for k in sd_a:
        assert torch.equal(sd_a[k], sd_b[k]), k
    return trainer2, module2


def wenzhong_recipe(tmp_path, min_drop, device):
    """finetune_wenzhong.py:37-140 in miniature: GPT2LMHeadModel.from_pretrained(dir), the compat GPT2QADataModel, a torch AdamW
    with name-based no-decay groups + linear warm-up returned in PL's list-of-dict form, default (DDP) strategy, a
    ModelCheckpoint whose file name formats a logged metric."""
    import argparse
    import pytorch_lightning as pl
    from pytorch_lightning import Trainer, loggers
    from pytorch_lightning.callbacks import ModelCheckpoint
    from transformers import GPT2Config, GPT2LMHeadModel
    from transformers.optimization import get_linear_schedule_with_warmup
    from fengshen.data.task_dataloader.medicalQADataset import GPT2QADataModel
    assert not GPT2LMHeadModel.__module__.startswith("transformers.")

    mdir = tmp_path / "m"
    F.gpt2_tokenizer_dir(mdir)
    F.qa_files(tmp_path / "data", n=48)
    GPT2LMHeadModel(GPT2Config(**{k: v for k, v in F.GPT2_CFG.items() if k != "model_type"})).save_pretrained(str(mdir))
    assert (mdir / "pytorch_model.bin").exists() and (mdir / "config.json").exists()

    class GPT2FinetuneMedicalQA(pl.LightningModule):
        def __init__(self, args, num_data):
            super().__init__()
            self.args, self.num_data = args, num_data
            self.model = GPT2LMHeadModel.from_pretrained(args.pretrained_model_path)

        def setup(self, stage) -> None:
            if stage == 'fit':
                num_gpus = self.trainer.gpus if self.trainer.gpus is not None else 0
                self.total_step = int(self.trainer.max_epochs * self.num_data
                                      / (max(1, num_gpus) * self.trainer.accumulate_grad_batches))

        def training_step(self, batch, batch_idx):
            output = self.model(input_ids=batch['input_ids'], attention_mask=batch['attention_mask'], labels=batch['labels'])
            self.log('train_loss', output.loss)
            return output.loss

        def configure_optimizers(self):
            no_decay = ['bias', 'LayerNorm.bias', 'LayerNorm.weight']
            paras = [(n, p) for n, p in self.named_parameters() if p.requires_grad]
            paras = [{'params': [p for n, p in paras if not any(nd in n for nd in no_decay)],
                      'weight_decay': self.args.weight_decay},
                     {'params': [p for n, p in paras if any(nd in n for nd in no_decay)], 'weight_decay': 0.0}]
            optimizer = torch.optim.AdamW(paras, lr=self.args.learning_rate)
            scheduler = get_linear_schedule_with_warmup(optimizer, int(self.total_step * self.args.warmup), self.total_step)
            return [{'optimizer': optimizer, 'lr_scheduler': {'scheduler': scheduler, 'interval': 'step', 'frequency': 1}}]

    p = argparse.ArgumentParser("QA Task")
    p.add_argument('--do_eval_only', action='store_true', default=False)
    p.add_argument('--pretrained_model_path', default='google/mt5-small', type=str)
    p = GPT2QADataModel.add_data_specific_args(p)
    p = Trainer.add_argparse_args(p)
    p.add_argument('--learning_rate', default=1e-4, type=float)
    p.add_argument('--weight_decay', default=0.1, type=float)
    p.add_argument('--warmup', default=0.01, type=float)
    args = p.parse_args(["--pretrained_model_path", str(mdir), "--data_dir", str(tmp_path / "data"), "--train_batchsize", "4",
                         "--valid_batchsize", "4", "--max_seq_length", "64", "--num_workers", "0", "--max_epochs", "2",
                         "--gpus", "1", "--learning_rate", "2e-3", "--warmup", "0.1", "--log_every_n_steps", "1",
                         "--default_root_dir", str(tmp_path)])
    data_model = GPT2QADataModel(args)
    model = GPT2FinetuneMedicalQA(args, len(data_model.train_dataloader()))
    ckpt = ModelCheckpoint(monitor='train_loss', save_top_k=3, mode='min', every_n_train_steps=10, save_weights_only=True,
                           dirpath=str(tmp_path / "ckpt"), filename='model-{epoch:02d}-{train_loss:.4f}', save_last=True)
    logger = loggers.TensorBoardLogger(save_dir=os.path.join(args.default_root_dir, 'log/'), name='WenZhong')
    trainer = Trainer.from_argparse_args(args, logger=logger, callbacks=[ckpt])
    trainer.fit(model, data_model)
    assert trainer.global_step == 24                                   # 48 rows / 4 per step x 2 epochs
    losses = losses_of(trainer)
    assert len(losses) == 24 and sum(losses[-3:]) / 3 < sum(losses[:3]) / 3 - min_drop, losses
    names = sorted(os.listdir(tmp_path / "ckpt"))
    assert "last.ckpt" in names and any(n.startswith("model-0") and "{" not in n for n in names), names
    assert (tmp_path / "ckpt" / "last.ckpt" / "checkpoint" / "mp_rank_00_model_states.pt").exists()
    assert not (tmp_path / "ckpt" / "last.ckpt" / "checkpoint" / "zero_pp_rank_0_mp_rank_00_optim_states.pt").exists()
    # padding really is excluded: the same batch with garbage under the padding gives the same loss
    b = next(iter(data_model.val_dataloader()))
    dev = lambda t: t.to(device)
    with torch.no_grad():
        l1 = model.model(input_ids=dev(b['input_ids']), attention_mask=dev(b['attention_mask']), labels=dev(b['labels'])).loss
        ids2 = torch.where(b['attention_mask'] == 0, torch.full_like(b['input_ids'], 7), b['input_ids'])
        l2 = model.model(input_ids=dev(ids2), attention_mask=dev(b['attention_mask']), labels=dev(b['labels'])).loss
    assert abs(float(l1) - float(l2)) < 1e-3
    return trainer, model


def t5_recipe(tmp_path, min_drop, lr="2e-3"):
    """pretrain_t5.py:16-155 in miniature (its `bert_tokenizer` branch: model from MT5Config, no pretrained weights): the compat
    UnsuperviseT5DataModel over a tokenised `datasets` directory (span corruption in the collate step, Megatron sampler), the
    module's own total-step arithmetic, fengshen.models.model_utils.configure_optimizers, on_save_checkpoint exporting
    `hf_pretrained_epoch{}_step{}` next to the checkpoints, then a resumed second epoch."""
    import argparse
    import pytorch_lightning as pl
    from pytorch_lightning import Trainer, loggers
    from pytorch_lightning.callbacks import LearningRateMonitor
    from transformers import MT5Config, MT5ForConditionalGeneration
    from fengshen.data.t5_dataloader.t5_datasets import UnsuperviseT5DataModel
    from fengshen.models.model_utils import add_module_args, configure_optimizers
    from fengshen.utils.universal_checkpoint import UniversalCheckpoint
    assert not MT5ForConditionalGeneration.__module__.startswith("transformers.")
    F.t5_dir(tmp_path / "m")
    F.t5_tokenised_dir(tmp_path / "tok")

    class MT5PretrainModel(pl.LightningModule):
        def __init__(self, args):
            super().__init__()
            self.save_hyperparameters(args)
            self.model = MT5ForConditionalGeneration(MT5Config.from_pretrained(args.pretrained_model_path))

        def setup(self, stage) -> None:
            if stage == 'fit':
                train_loader = self.trainer._data_connector._train_dataloader_source.dataloader()
                tb_size = self.hparams.train_batchsize * max(1, self.trainer.world_size)
                ab_size = self.trainer.accumulate_grad_batches * float(self.trainer.max_epochs)
                self.total_steps = (len(train_loader.dataset) * self.trainer.max_epochs // tb_size) // ab_size

        def configure_optimizers(self):
            return configure_optimizers(self)

        def training_step(self, batch, batch_idx):
            output = self.model(input_ids=batch['input_ids'], labels=batch['labels'])
            y_pred = torch.argmax(output.logits, dim=-1).view(size=(-1,))
            y_true = batch['labels'].view(size=(-1,)).float()
            self.log('train_loss', output.loss, sync_dist=True)
            self.log('train_acc', torch.sum(torch.eq(y_pred, y_true).float()) / y_true.shape[0], sync_dist=True)
            return output.loss

        def on_save_checkpoint(self, checkpoint) -> None:
            if self.trainer.global_rank == 0 and self.trainer.global_step % self.hparams.every_n_train_steps == 0:
                self.model.save_pretrained(os.path.join(
                    self.trainer.checkpoint_callback.dirpath,
                    'hf_pretrained_epoch{}_step{}'.format(self.trainer.current_epoch, self.trainer.global_step)))

        def on_load_checkpoint(self, checkpoint) -> None:
            if 'global_samples' in checkpoint:
                self.consumed_samples = checkpoint['global_samples']
            self.trainer.fit_loop.epoch_loop._batches_that_stepped = checkpoint["global_step"]

    def run(max_steps):
        p = argparse.ArgumentParser("Pretrain Unsupervise.")
        p.add_argument('--pretrained_model_path', default=None, type=str)
        p.add_argument('--new_vocab_path', default=None, type=str)
        p.add_argument('--max_seq_length', default=1024, type=int)
        p.add_argument('--ckpt_path', default=None, type=str)
        p = add_module_args(p)       # the flags model_utils.configure_optimizers reads (the reference script omits this call)
        p = UnsuperviseT5DataModel.add_data_specific_args(p)
        p = Trainer.add_argparse_args(p)
        p = UniversalCheckpoint.add_argparse_args(p)
        args = p.parse_args(["--pretrained_model_path", str(tmp_path / "m"), "--tokenizer_type", "bert_tokenizer",
                             "--train_data_path", str(tmp_path / "tok"), "--train_split_size", "0.999", "--max_seq_length", "64",
                             "--train_batchsize", "4", "--valid_batchsize", "4", "--dataloader_num_workers", "0",
                             "--max_epochs", "1", "--max_steps", str(max_steps), "--learning_rate", lr, "--warmup_ratio", "0.1",
                             "--strategy", "deepspeed_stage_2", "--log_every_n_steps", "1", "--default_root_dir", str(tmp_path),
                             "--save_ckpt_path", str(tmp_path / "ckpt"), "--load_ckpt_path", str(tmp_path / "ckpt" / "last.ckpt"),
                             "--every_n_train_steps", "6", "--save_last", "--precision", "bf16"])
        data_model = UnsuperviseT5DataModel(args)
        assert (data_model.expanded_inputs_length, data_model.targets_length) == (70, 14)
        model = MT5PretrainModel(args)
        logger = loggers.TensorBoardLogger(save_dir=os.path.join(args.default_root_dir, 'logs/'))
        trainer = Trainer.from_argparse_args(args, logger=logger,
                                             callbacks=[UniversalCheckpoint(args), LearningRateMonitor(logging_interval='step')])
        trainer.fit(model, data_model, ckpt_path=args.load_ckpt_path)
        return trainer, model, data_model

    trainer, model, dm = run(6)                                                  # half of the epoch (48 chunks / 4 = 12 steps)
    assert trainer.global_step == 6 and trainer.engine.stage == 2
    losses = losses_of(trainer)
    assert len(losses) == 6 and all(l == l for l in losses)
    if min_drop is not None:
        assert sum(losses[-2:]) / 2 < sum(losses[:2]) / 2 - min_drop, losses
    batch = next(iter(dm.val_dataloader()))
    assert batch["input_ids"].shape == (4, 64) and batch["labels"].shape == (4, 14)
    assert (batch["input_ids"][:, -1] == 1).all() and (batch["input_ids"] >= 512 - 8).any()      # EOS last, sentinels present
    exported = sorted(d for d in os.listdir(tmp_path / "ckpt") if d.startswith("hf_pretrained"))
    assert exported == ["hf_pretrained_epoch0_step6"], exported
    again = MT5ForConditionalGeneration.from_pretrained(str(tmp_path / "ckpt" / exported[0]))
    assert torch.equal(again.state_dict()["shared.weight"], model.model.state_dict()["shared.weight"])
    # the rest of the epoch from last.ckpt: the Megatron sampler continues behind the 24 consumed chunks
    seen = []
    orig = UnsuperviseT5DataModel.collate_fn
    UnsuperviseT5DataModel.collate_fn = lambda self, ex: (seen.append([e["input_ids"][:4] for e in ex]), orig(self, ex))[1]
    try:
        trainer2, model2, dm2 = run(-1)
    finally:
        UnsuperviseT5DataModel.collate_fn = orig
    assert trainer2.global_step == 12 and model2.consumed_samples == 24
    assert len(seen) == 6 and seen[0][0] == dm2.train_dataset[24]["input_ids"][:4]
    return trainer2, model2
