"""UniversalDataModule — flags, constructor and sampler selection of
fengshen/data/universal_datamodule/universal_datamodule.py:20-160. `datasets` may be passed in directly (the documented
escape hatch at :52-55); loading corpora by name needs the reference's private fs_datasets and is not reproduced."""
from pytorch_lightning import LightningDataModule
from torch.utils.data import DataLoader, DistributedSampler

from fengshen.models.megatron import mpu


def get_consume_samples(data_model):
    """universal_datamodule.py:8-17."""
    if hasattr(data_model.trainer.lightning_module, 'consumed_samples'):
        consumed_samples = data_model.trainer.lightning_module.consumed_samples
        print('get consumed samples from model: {}'.format(consumed_samples))
    else:
        world_size = data_model.trainer.world_size
        consumed_samples = max(0, data_model.trainer.global_step - 1) * \
            data_model.hparams.train_batchsize * world_size * data_model.trainer.accumulate_grad_batches
        print('calculate consumed samples: {}'.format(consumed_samples))
    return consumed_samples


class UniversalDataModule(LightningDataModule):
    # (flag, add_argument keywords) — universal_datamodule.py:22-46: the schema the launch scripts pass
    _FLAGS = (
        ('--num_workers', dict(default=8, type=int)),
        ('--dataloader_workers', dict(default=2, type=int)),
        ('--train_batchsize', dict(default=16, type=int)),
        ('--val_batchsize', dict(default=16, type=int)),
        ('--test_batchsize', dict(default=16, type=int)),
        ('--datasets_name', dict(type=str, default=None)),
        ('--train_datasets_field', dict(type=str, default='train')),
        ('--val_datasets_field', dict(type=str, default='validation')),
        ('--test_datasets_field', dict(type=str, default='test')),
        ('--train_file', dict(type=str, default=None)),
        ('--val_file', dict(type=str, default=None)),
        ('--test_file', dict(type=str, default=None)),
        ('--raw_file_type', dict(type=str, default='json')),
        ('--sampler_type', dict(type=str, choices=['single', 'random'], default='random')),
        ('--use_mpu', dict(action="store_true", default=False)),
    )

    @staticmethod
    def add_data_specific_args(parent_args):
        group = parent_args.add_argument_group('Universal DataModule')
        for flag, kw in UniversalDataModule._FLAGS:
            group.add_argument(flag, **kw)
        return parent_args

    def __init__(self, tokenizer, collate_fn, args, datasets=None, **kwargs):
        super().__init__()
        if datasets is not None:
            self.datasets = datasets
        elif getattr(args, 'datasets_name', None) is not None:
            raise NotImplementedError("fsb200 compat: loading IDEA corpora by name needs fengshen.data.fs_datasets "
                                      "(private data, out of scope); pass `datasets=` or --train_file")
        else:
            from datasets import load_dataset
            self.datasets = load_dataset(args.raw_file_type, data_files={
                args.train_datasets_field: args.train_file, args.val_datasets_field: args.val_file,
                args.test_datasets_field: args.test_file})
        self.tokenizer = tokenizer
        self.collate_fn = collate_fn
        self.save_hyperparameters(args)

    def get_custom_sampler(self, ds):
        from .universal_sampler import PretrainingRandomSampler, PretrainingSampler
        world_size = self.trainer.world_size
        consumed_samples = get_consume_samples(self)
        rank = mpu.get_data_parallel_rank() if self.hparams.use_mpu else self.trainer.global_rank
        size = mpu.get_data_parallel_world_size() if self.hparams.use_mpu else world_size
        if self.hparams.sampler_type == 'random':
            return PretrainingRandomSampler(total_samples=len(ds), consumed_samples=consumed_samples,
                                            micro_batch_size=self.hparams.train_batchsize, data_parallel_rank=rank,
                                            data_parallel_size=size, epoch=self.trainer.current_epoch)
        if self.hparams.sampler_type == 'single':
            return PretrainingSampler(total_samples=len(ds), consumed_samples=consumed_samples,
                                      micro_batch_size=self.hparams.train_batchsize, data_parallel_rank=rank,
                                      data_parallel_size=size)
        raise Exception('Unknown sampler type: {}'.format(self.hparams.sampler_type))

    def setup(self, stage=None):
        return

    def _loader(self, ds, batch_size, custom_sampler, data_parallel=False):
        collate_fn = getattr(ds, 'collate_fn', self.collate_fn)
        workers = getattr(self.hparams, 'dataloader_workers', 0)
        if custom_sampler:
            return DataLoader(ds, batch_sampler=self.get_custom_sampler(ds), num_workers=workers, collate_fn=collate_fn,
                              pin_memory=True)
        sampler = None
        if self.trainer is not None and self.trainer.world_size > 1:
            # data_parallel: shard over the data-parallel group, so that the ranks of one tensor-parallel group read the same
            # batch (without tensor parallelism that group is the whole world)
            rank = mpu.get_data_parallel_rank() if data_parallel else self.trainer.global_rank
            size = mpu.get_data_parallel_world_size() if data_parallel else self.trainer.world_size
            sampler = DistributedSampler(ds, num_replicas=size, rank=rank, shuffle=False)
        return DataLoader(ds, batch_size=batch_size, sampler=sampler, num_workers=workers, collate_fn=collate_fn,
                          pin_memory=True)

    def train_dataloader(self):
        ds = self.datasets[self.hparams.train_datasets_field]
        return self._loader(ds, self.hparams.train_batchsize, self.hparams.get('replace_sampler_ddp', True) is False)

    def val_dataloader(self):
        ds = self.datasets[self.hparams.val_datasets_field]
        return self._loader(ds, self.hparams.val_batchsize, False, data_parallel=True)

    def test_dataloader(self):
        ds = self.datasets[self.hparams.test_datasets_field]
        return self._loader(ds, self.hparams.test_batchsize, False)

    def predict_dataloader(self):
        return self.test_dataloader()
