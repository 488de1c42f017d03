"""Ziya-LLaMA random-init pretraining step, written against the REFERENCE's import surface only
(fengshen.*, pytorch_lightning, deepspeed) — the structure of fengshen/examples/ziya_llama/finetune_ziya_llama.py:88-227
with the model built from a config instead of `from_pretrained` (SURVEY.md §0 fact 5) and a synthetic token dataset
(BASELINE.json metric: synthetic token batches). Run with fengshen-lm_b200/compat and fengshen-lm_b200 on PYTHONPATH:

  PYTHONPATH=fengshen-lm_b200/compat:fengshen-lm_b200 python examples/pretrain_ziya_llama.py \
      --hidden_size 512 --num_layers 4 --num_heads 8 --vocab_size 4096 --max_seq_length 256 \
      --train_batchsize 4 --max_steps 20 --learning_rate 1e-3 --adam_beta2 0.95 --strategy deepspeed_stage_2

Multi-GPU: launch under `python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 ...`.
"""
import argparse
import os

import torch
import pytorch_lightning as pl
from pytorch_lightning.callbacks import LearningRateMonitor
from pytorch_lightning.loggers import WandbLogger
from fengshen.models.model_utils import (
    configure_optimizers,
    add_module_args,
    get_total_steps
)
from fengshen.models.llama.modeling_llama import LlamaForCausalLM
from fengshen.models.llama.configuration_llama import LlamaConfig
from fengshen.models.megatron import mpu
from fengshen.data.universal_datamodule import UniversalDataModule
from fengshen.utils.universal_checkpoint import UniversalCheckpoint
from fengshen.strategies.megatron_deepspeed import DeepSpeedStrategy


class SyntheticTokens(torch.utils.data.Dataset):
    """Seeded uniform token ids, one sample = one sequence (SURVEY.md §8d)."""

    def __init__(self, vocab_size, seq_len, n, seed=1234):
        g = torch.Generator().manual_seed(seed)
        self.ids = torch.randint(0, vocab_size, (n, seq_len), generator=g, dtype=torch.int64)

    def __len__(self):
        return self.ids.shape[0]

    def __getitem__(self, i):
        return self.ids[i]


class SyntheticCollator:
    """Emits the keys of LlamaSFTCollator (finetune_ziya_llama.py:79-84): input_ids, attention_mask, labels, position_ids."""

    def __call__(self, samples):
        ids = torch.stack(samples)
        return {"input_ids": ids, "attention_mask": torch.ones_like(ids), "labels": ids.clone(),
                "position_ids": torch.arange(ids.shape[1], dtype=torch.int64)[None].expand_as(ids).contiguous()}


class Llama(pl.LightningModule):
    @staticmethod
    def add_module_specific_args(parent_parser):
        parser = parent_parser.add_argument_group('ziya_llama pretrain')
        parser.add_argument('--max_seq_length', type=int, default=1024)
        parser.add_argument('--model_parallel_size', type=int, default=1)
        parser.add_argument('--hidden_size', type=int, default=5120)
        parser.add_argument('--num_layers', type=int, default=40)
        parser.add_argument('--num_heads', type=int, default=40)
        parser.add_argument('--vocab_size', type=int, default=39424)
        parser.add_argument('--num_samples', type=int, default=4096)
        parser.add_argument('--gradient_checkpointing', action='store_true',
                            help='recompute each layer in the backward instead of keeping its activations')
        return parent_parser

    def __init__(self, args):
        super().__init__()
        self.save_hyperparameters(args)

    def setup(self, stage) -> None:
        assert mpu.get_model_parallel_world_size() == 1
        config = LlamaConfig(vocab_size=self.hparams.vocab_size, hidden_size=self.hparams.hidden_size,
                             num_hidden_layers=self.hparams.num_layers, num_attention_heads=self.hparams.num_heads)
        self.model = LlamaForCausalLM(config).cuda()
        if self.hparams.gradient_checkpointing:
            self.model.gradient_checkpointing_enable()
        if stage == 'fit':
            self.total_steps = get_total_steps(self.trainer, self.hparams)
            print('Total steps: {}'.format(self.total_steps))

    def configure_optimizers(self):
        return configure_optimizers(self)

    def forward(self, **batch):
        return self.model(**batch)

    def training_step(self, batch, batch_idx):
        output = self(**batch)
        self.log('train/loss', output.loss, sync_dist=True)
        return output.loss

    def on_load_checkpoint(self, checkpoint) -> None:
        if 'global_samples' in checkpoint:
            self.consumed_samples = checkpoint['global_samples']


def main(argv=None):
    args_parser = argparse.ArgumentParser()
    args_parser.add_argument('--wandb_project', type=str, default="ziya_llama13b_pretrain_example")
    args_parser.add_argument('--wandb_name', type=str, default="exp1")
    args_parser = add_module_args(args_parser)
    args_parser = pl.Trainer.add_argparse_args(args_parser)
    args_parser = UniversalDataModule.add_data_specific_args(args_parser)
    args_parser = Llama.add_module_specific_args(args_parser)
    args_parser = UniversalCheckpoint.add_argparse_args(args_parser)
    args = args_parser.parse_args(argv)

    datasets = {"train": SyntheticTokens(args.vocab_size, args.max_seq_length, args.num_samples)}
    data_module = UniversalDataModule(tokenizer=None, args=args, collate_fn=SyntheticCollator(), datasets=datasets)
    model = Llama(args)
    strategy = DeepSpeedStrategy(
        tensor_model_parallel_size=args.model_parallel_size,
        pipe_model_parallel_size=1,
        mpu_seed=42,
    )
    if args.load_ckpt_path is not None and not os.path.exists(args.load_ckpt_path):
        print('--------warning no checkpoint found--------, remove args')
        args.load_ckpt_path = None
    wandb_logger = WandbLogger(project=args.wandb_project, name=args.wandb_name, save_dir=args.default_root_dir)
    lr_monitor = LearningRateMonitor(logging_interval='step')
    checkpoint_callback = UniversalCheckpoint(args)
    trainer = pl.Trainer.from_argparse_args(args, strategy=strategy, logger=wandb_logger,
                                            callbacks=[lr_monitor, checkpoint_callback])
    trainer.fit(model, data_module, ckpt_path=args.load_ckpt_path)
    return trainer, model


if __name__ == '__main__':
    main()
