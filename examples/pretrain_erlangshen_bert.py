"""Erlangshen-MegatronBERT pretraining (masked LM + sentence order) on fsb200, written against the REFERENCE's import surface
only: the transformers class names, pytorch_lightning, fengshen.data / fengshen.models.model_utils / fengshen.utils. It plays the
role of fengshen/examples/pretrain_erlangshen_bert/pretrain_erlangshen.py (same command-line flags, same LightningModule hooks,
same recipe) for machines that do not hold the reference tree; the collator comes from the library
(fengshen.data.data_utils.collators) and the corpus is a JSON-lines file ({"text": ...} per line) handed to UniversalDataModule
through its `datasets=` argument.

  PYTHONPATH=fengshen-lm_b200 python -m fsb200.launch examples/pretrain_erlangshen_bert.py \
      --model_path <dir with config.json + vocab.txt> --train_file corpus.json --train_batchsize 32 --max_seq_length 512 \
      --max_epochs 1 --strategy deepspeed_stage_1 --replace_sampler_ddp False --learning_rate 1e-4

`fsb200.launch` puts the compat packages on sys.path and binds `transformers.MegatronBertForPreTraining` to the fsb200-backed
class. The recipe's DeepSpeed JSON (ZeRO stage, gradient_clipping) is read from $PL_DEEPSPEED_CONFIG_PATH as in the reference
(pretrain_erlangshen_base.sh:24-39). Dropout must be 0 in config.json: fsb200 rejects dropout > 0 loudly.

--pack_sequences (off by default) wraps the collator, Python or --native_collator, in fsb200.packing.MLMPackingCollator: the
documents of a batch are packed whole into rows of --max_seq_length instead of one padded document per row, and
`forward(**batch)` hands the packed keys (segment_ids, position_ids, cls_positions) to the model.

--fp8 (off by default) builds the model with `fp8=True`: each layer's four projections train in FP8 (e4m3 activations and
weights, e5m2 gradients, per-tensor scales); the weights, gradients, optimizer state and checkpoints stay as without it."""
import argparse
import json
import os

import torch
from pytorch_lightning import LightningModule, Trainer
from pytorch_lightning.callbacks import LearningRateMonitor
from pytorch_lightning.loggers import TensorBoardLogger
from transformers import AutoTokenizer, MegatronBertConfig, MegatronBertForPreTraining

from fengshen.data.data_utils.collators import ErLangShenCollator, FastErLangShenCollator
from fengshen.data.universal_datamodule import UniversalDataModule
from fengshen.models.model_utils import add_module_args, configure_optimizers, get_total_steps
from fengshen.utils.universal_checkpoint import UniversalCheckpoint


class JsonLines(torch.utils.data.Dataset):
    """One JSON object per line, kept in memory."""

    def __init__(self, path):
        with open(path, encoding="utf8") as fh:
            self.rows = [json.loads(line) for line in fh if line.strip()]

    def __getitem__(self, i):
        return self.rows[i]

    def __len__(self):
        return len(self.rows)


class ErLangShenBert(LightningModule):
    """The module of pretrain_erlangshen.py:126-197 by its hooks: model from `--model_path/config.json` (random init), optimizer
    and schedule from fengshen.models.model_utils, loss = MLM + sentence order, masked-token accuracy logged next to it, the sample
    counter restored from a checkpoint for the resumable sampler."""

    @staticmethod
    def add_module_specific_args(parent_parser):
        group = parent_parser.add_argument_group('Erlangshen Bert')
        for flag, typ, default in (('--masked_lm_prob', float, 0.15), ('--max_seq_length', int, 512),
                                   ('--sample_content_key', str, 'text')):
            group.add_argument(flag, type=typ, default=default)
        return parent_parser

    def __init__(self, args, tokenizer, **_):
        super().__init__()
        self.save_hyperparameters(args)
        self.tokenizer = tokenizer
        self.config = MegatronBertConfig.from_pretrained(args.model_path)
        # fp8 is an fsb200 keyword: pass it only when asked, so that the default build is the reference's call
        self.model = (MegatronBertForPreTraining(self.config, fp8=True) if getattr(args, 'fp8', False)
                      else MegatronBertForPreTraining(self.config))

    def setup(self, stage):
        if stage == 'fit':
            self.total_steps = get_total_steps(self.trainer, self.hparams)
            print(f'Total steps: {self.total_steps}')

    def configure_optimizers(self):
        return configure_optimizers(self)

    def forward(self, **batch):
        return self.model(**batch)

    @staticmethod
    def masked_accuracy(logits, labels):
        """Share of masked positions whose arg-max is the original token."""
        picked = labels != -100
        hits = (logits[picked].argmax(dim=-1) == labels[picked]).float().sum()
        return hits / picked.sum().clamp(min=1)

    def training_step(self, batch, batch_idx):
        out = self(**batch)
        self.log('train_loss', out.loss, sync_dist=True)
        self.log('train_acc', self.masked_accuracy(out.prediction_logits, batch['labels']), sync_dist=True)
        return out.loss

    def on_load_checkpoint(self, checkpoint):
        self.trainer.fit_loop.epoch_loop._batches_that_stepped = checkpoint["global_step"]
        if 'global_samples' in checkpoint:
            self.consumed_samples = checkpoint['global_samples']


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    parser.add_argument('--native_collator', action='store_true', default=False,
                        help='assemble and mask the samples in libfsb200.so (fsb_bert_collate): same batches, ~1000x less host time')
    parser.add_argument('--pack_sequences', action='store_true', default=False,
                        help='pack the documents of each batch whole into rows of max_seq_length (fsb200.packing)')
    parser.add_argument('--fp8', action='store_true', default=False,
                        help="train the layer projections in FP8 (fsb200's MegatronBertForPreTraining(config, fp8=True))")
    for add in (add_module_args, UniversalDataModule.add_data_specific_args, Trainer.add_argparse_args,
                ErLangShenBert.add_module_specific_args, UniversalCheckpoint.add_argparse_args):
        parser = add(parser)
    args = parser.parse_args(argv)
    if args.load_ckpt_path is not None and not os.path.exists(args.load_ckpt_path):
        print('--------warning no checkpoint found--------, remove args')
        args.load_ckpt_path = None
    return args


def build_data(args, tokenizer):
    collator_cls = FastErLangShenCollator if args.native_collator else ErLangShenCollator
    collator = collator_cls(tokenizer=tokenizer, max_seq_length=args.max_seq_length, masked_lm_prob=args.masked_lm_prob,
                            content_key=args.sample_content_key)
    collator.setup()
    if args.pack_sequences:
        from fsb200.packing import MLMPackingCollator
        collator = MLMPackingCollator(collator, args.max_seq_length, tokenizer.pad_token_id)
    return UniversalDataModule(tokenizer=tokenizer, args=args, collate_fn=collator,
                               datasets={args.train_datasets_field: JsonLines(args.train_file)})


def main(argv=None):
    args = parse_args(argv)
    tokenizer = AutoTokenizer.from_pretrained(args.model_path)
    data_module = build_data(args, tokenizer)
    module = ErLangShenBert(args, tokenizer=tokenizer)
    logger = TensorBoardLogger(save_dir=os.path.join(args.default_root_dir or ".", 'logs'), name='erlangshen')
    trainer = Trainer.from_argparse_args(args, logger=logger,
                                         callbacks=[LearningRateMonitor(logging_interval='step'), UniversalCheckpoint(args)])
    trainer.fit(module, data_module, ckpt_path=args.load_ckpt_path)
    return trainer, module


if __name__ == '__main__':
    main()
