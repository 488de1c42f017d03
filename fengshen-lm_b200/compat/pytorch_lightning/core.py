import argparse
import random

import numpy as np
import torch
from torch import nn


class _HParams(dict):
    """Attribute + item access, like PL's AttributeDict."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


class _HParamsMixin:
    def save_hyperparameters(self, *args, **kwargs):
        hp = _HParams()
        for a in args:
            if isinstance(a, argparse.Namespace):
                hp.update(vars(a))
            elif isinstance(a, dict):
                hp.update(a)
        hp.update(kwargs)
        object.__setattr__(self, "_hparams", hp)

    @property
    def hparams(self):
        if not hasattr(self, "_hparams"):
            object.__setattr__(self, "_hparams", _HParams())
        return self._hparams


class LightningModule(_HParamsMixin, nn.Module):
    def __init__(self):
        super().__init__()
        self.trainer = None
        self._logged = {}

    # ---- hooks the example scripts override
    def setup(self, stage=None):
        pass

    def configure_optimizers(self):
        raise NotImplementedError

    def training_step(self, batch, batch_idx):
        raise NotImplementedError

    def validation_step(self, batch, batch_idx):
        pass

    def predict_step(self, batch, batch_idx):
        pass

    def on_load_checkpoint(self, checkpoint):
        pass

    def on_save_checkpoint(self, checkpoint):
        pass

    # ---- services
    def log(self, name, value, sync_dist=False, **_):
        if self.trainer is not None and getattr(self.trainer, "_val_acc", None) is not None:
            # inside a validation run: the run's batch-size-weighted mean, reported when the run ends
            self.trainer._log_val(name, value, sync_dist, self.device)
            return
        if isinstance(value, torch.Tensor):
            value = value.detach()
            if sync_dist and self.trainer is not None and self.trainer.world_size > 1:
                import torch.distributed as dist
                value = value.clone()
                dist.all_reduce(value, op=dist.ReduceOp.SUM)
                value = value / self.trainer.world_size
        self._logged[name] = value
        if self.trainer is not None:
            self.trainer.callback_metrics[name] = value

    def log_dict(self, d, **kw):
        for k, v in d.items():
            self.log(k, v, **kw)

    @property
    def device(self):
        for p in self.parameters():
            return p.device
        return torch.device("cpu")

    @property
    def global_rank(self):
        return 0 if self.trainer is None else self.trainer.global_rank

    @property
    def global_step(self):
        return 0 if self.trainer is None else self.trainer.global_step

    @property
    def current_epoch(self):
        return 0 if self.trainer is None else self.trainer.current_epoch


class LightningDataModule(_HParamsMixin):
    def __init__(self):
        self.trainer = None

    def prepare_data(self):
        pass

    def setup(self, stage=None):
        pass

    def train_dataloader(self):
        return None

    def val_dataloader(self):
        return None

    def test_dataloader(self):
        return None

    def predict_dataloader(self):
        return None


def seed_everything(seed, workers=False):
    random.seed(seed)
    np.random.seed(seed % (2 ** 32))
    torch.manual_seed(seed)
    return seed
