"""`pl.Trainer` for the hot-path example scripts, executing the step with fsb200 (model kernels + ZeroEngine).

Surface kept (SURVEY.md §8b): `add_argparse_args`, `from_argparse_args`, `fit`, `predict`, `save_checkpoint`; attributes
`max_epochs, max_steps, world_size, global_rank, accumulate_grad_batches, gpus, global_step, current_epoch, strategy,
checkpoint_callback, lightning_module, optimizers, callback_metrics`, and the two private paths the reference pokes:
`_data_connector._train_dataloader_source.dataloader()` (fengshen/models/model_utils.py:195) and
`fit_loop.epoch_loop._batches_that_stepped` (examples/pretrain_erlangshen_bert/pretrain_erlangshen.py:197).

Validation inside `fit` restates PyTorch-Lightning 1.9 (the names in brackets are PL 1.9's, to check against an install):
- Enabled (`Trainer.enable_validation`) only when the module overrides `validation_step` (`is_overridden`), a validation
  loader exists (`datamodule.val_dataloader()` or `fit(val_dataloaders=...)`) and `limit_val_batches` is not 0. Otherwise
  `fit` runs exactly as without validation, and `val_dataloader()` is never called. An error it raises propagates.
- Cadence (`Trainer.val_check_batch`, `TrainingEpochLoop._should_check_val_fx`): a float `val_check_interval` f gives
  `val_check_batch = max(1, int(n_train_batches * f))`, an int N gives N. An int above the epoch's batch count is a
  `ValueError` unless `check_val_every_n_epoch` is None; a float with `check_val_every_n_epoch=None` is a `ValueError`
  (PL's "should be an integer"). After training batch i, validation runs when
  `(i + 1) % val_check_batch == 0`, where i is the batch index within the epoch, or the total batch index across epochs
  when `check_val_every_n_epoch` is None (`total_batch_idx`). Batches are micro-batches, so a run may fall inside a
  gradient-accumulation window. Only epochs with `(epoch + 1) % check_val_every_n_epoch == 0` validate
  (`_should_check_val_epoch`).
- Limits (`_parse_num_batches`): `limit_val_batches` is a fraction (float) or a count (int) of the loader's batches; a
  fraction that leaves 0 batches of a non-empty loader is a `ValueError`; an empty loader means no validation. `num_sanity_val_steps` (default 2, -1 = all) batches run once before
  the first training batch, also on resume (`_run_sanity_check`); their metrics are discarded.
- Each run: `module.eval()`, `torch.no_grad()`, `validation_step(batch, batch_idx)` with batch_idx counted within the run,
  then `module.train()`. PL wraps only the sanity pass in `isolate_rng`; here every run is, so that a validation run
  leaves the training run bit-for-bit unchanged even when a collator draws random numbers.
- Metrics (`ResultCollection`, `on_epoch=True`, mean reduction): `LightningModule.log` inside a run accumulates the
  batch-size-weighted mean, the batch size being dim 0 of the batch's first tensor (`extract_batch_size`). `sync_dist=True`
  makes it the global weighted mean (one all-reduce per metric per run). The result goes to `callback_metrics` and, from
  rank 0, to the logger once at `step = global_step`; training log lines carry training metrics only.
"""
import argparse
import os
import random
from types import SimpleNamespace

import numpy as np
import torch
import torch.distributed as dist

from .callbacks import ModelCheckpoint
from .core import LightningModule
from .strategies import DDPStrategy, DeepSpeedStrategy, strategy_from_string


def _int_or_float(x):
    """PL's `_int_or_float_type` (utilities/argparse.py): '100' is the int 100, '0.1' and '1.0' are floats."""
    return float(x) if "." in str(x) else int(x)


def _batch_limit(v, name):
    """PL's `_determine_batch_limits`: None -> 1.0; a value in [0, 1] keeps its type; a whole float above 1 becomes an int."""
    if v is None:
        return 1.0
    if 0 <= v <= 1:
        return v
    if v > 1 and v % 1.0 == 0:
        return int(v)
    raise ValueError(f"{name}={v!r}: expected a float in [0.0, 1.0] or an int >= 0")


_ARGS = [  # the PL-1.x Trainer flags that the reference's launch scripts pass (examples/*/*.sh)
    ("--max_epochs", int, None), ("--max_steps", int, -1), ("--gpus", int, None), ("--devices", int, None),
    ("--num_nodes", int, 1), ("--strategy", str, None), ("--precision", str, "32"),
    ("--accumulate_grad_batches", int, 1), ("--gradient_clip_val", float, None), ("--default_root_dir", str, None),
    ("--val_check_interval", _int_or_float, None), ("--check_val_every_n_epoch", int, 1), ("--log_every_n_steps", int, 50),
    ("--limit_val_batches", _int_or_float, None), ("--num_sanity_val_steps", int, 2), ("--accelerator", str, None),
    ("--resume_from_checkpoint", str, None), ("--enable_progress_bar", bool, True), ("--amp_backend", str, None),
    ("--profiler", str, None),
]


class Trainer:
    @classmethod
    def add_argparse_args(cls, parent_parser):
        g = parent_parser.add_argument_group("pl.Trainer")
        for flag, typ, default in _ARGS:
            if typ is bool:
                g.add_argument(flag, type=lambda s: str(s).lower() in ("1", "true", "yes"), default=default)
            else:
                g.add_argument(flag, type=typ, default=default)
        g.add_argument("--replace_sampler_ddp", type=lambda s: str(s).lower() in ("1", "true", "yes"), default=True)
        return parent_parser

    @classmethod
    def from_argparse_args(cls, args, **kwargs):
        known = {flag.lstrip("-") for flag, _, _ in _ARGS} | {"replace_sampler_ddp"}
        params = {k: v for k, v in vars(args).items() if k in known}
        params.update(kwargs)
        return cls(**params)

    def __init__(self, max_epochs=None, max_steps=-1, gpus=None, devices=None, num_nodes=1, strategy=None,
                 precision="32", accumulate_grad_batches=1, gradient_clip_val=None, default_root_dir=None,
                 logger=None, callbacks=None, log_every_n_steps=50, replace_sampler_ddp=True,
                 resume_from_checkpoint=None, val_check_interval=None, check_val_every_n_epoch=1,
                 limit_val_batches=None, num_sanity_val_steps=2, **_):
        self.max_epochs = max_epochs if max_epochs is not None else (1000 if (max_steps or -1) < 0 else -1)
        self.max_steps = max_steps if max_steps is not None else -1
        self.gpus = gpus if gpus is not None else devices
        self.num_nodes = num_nodes
        self.precision = str(precision)
        self.accumulate_grad_batches = int(accumulate_grad_batches or 1)
        self.gradient_clip_val = gradient_clip_val
        self.default_root_dir = default_root_dir or os.getcwd()
        self.logger = logger
        self.callbacks = list(callbacks or [])
        self.log_every_n_steps = log_every_n_steps
        self.replace_sampler_ddp = replace_sampler_ddp
        self.resume_from_checkpoint = resume_from_checkpoint   # PL-1.x flag: same meaning as fit(ckpt_path=...)
        self.val_check_interval = _batch_limit(val_check_interval, "val_check_interval")
        self.limit_val_batches = _batch_limit(limit_val_batches, "limit_val_batches")
        self.check_val_every_n_epoch = check_val_every_n_epoch
        self.num_sanity_val_steps = int(num_sanity_val_steps)
        self.val_check_batch = None       # set by fit() when validation is enabled
        self.sanity_checking = False
        self._val_acc = None              # name -> [device tensor (sum of v * batch size, sum of batch size), sync_dist]
        self._val_batch_size = 0
        self._val_names = set()           # metric names produced by validation, kept out of the training log lines
        if isinstance(strategy, str) or strategy is None:
            strategy = strategy_from_string(strategy)
        self.strategy = strategy
        self.world_size = int(os.environ.get("WORLD_SIZE", "1"))
        self.global_rank = int(os.environ.get("RANK", "0"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        self.global_step = 0
        self.current_epoch = 0
        self.just_stepped = False
        self.callback_metrics = {}
        self.optimizers, self.lr_scheduler_configs = [], []
        self.lightning_module, self.datamodule, self.engine = None, None, None
        self.fit_loop = SimpleNamespace(epoch_loop=SimpleNamespace(_batches_that_stepped=0))
        self._data_connector = SimpleNamespace(_train_dataloader_source=SimpleNamespace(dataloader=self._train_dl))
        self._train_loader = None

    # ---- plumbing ------------------------------------------------------------------------------------------------
    @property
    def checkpoint_callback(self):
        for c in self.callbacks:
            if isinstance(c, ModelCheckpoint):
                return c
        return None

    def _train_dl(self):
        if self._train_loader is None:
            self._train_loader = self.datamodule.train_dataloader()
        return self._train_loader

    def _setup_environment(self):
        if self.world_size > 1 and not dist.is_initialized():
            if not torch.cuda.is_available():
                dist.init_process_group("gloo")
            else:
                torch.cuda.set_device(self.local_rank)
                dist.init_process_group("nccl", device_id=torch.device("cuda", self.local_rank))
        elif torch.cuda.is_available():
            torch.cuda.set_device(self.local_rank)
        setup_mpu = getattr(self.strategy, "setup_mpu", None)
        if setup_mpu is not None:
            setup_mpu(self)

    @staticmethod
    def _find_fsb_model(module):
        for m in module.modules():
            if hasattr(m, "flat") and hasattr(m, "grad_hook"):
                return m
        raise RuntimeError("fsb200 Trainer: the LightningModule holds no fsb200 model (expected e.g. "
                           "fengshen.models.llama.modeling_llama.LlamaForCausalLM from the compat package)")

    def _unpack_optimizers(self, conf):
        opts, scheds = [], []
        if isinstance(conf, dict):
            conf = [conf]
        if isinstance(conf, (list, tuple)) and len(conf) == 2 and isinstance(conf[0], (list, tuple)):
            opts = list(conf[0])
            scheds = [s if isinstance(s, dict) else {"scheduler": s, "interval": "epoch"} for s in conf[1]]
        else:
            for c in (conf if isinstance(conf, (list, tuple)) else [conf]):
                if isinstance(c, dict):
                    opts.append(c["optimizer"])
                    if "lr_scheduler" in c:
                        s = c["lr_scheduler"]
                        scheds.append(s if isinstance(s, dict) else {"scheduler": s, "interval": "epoch"})
                else:
                    opts.append(c)
        return opts, scheds

    @staticmethod
    def _to_device(batch, device):
        return {k: (v.to(device, non_blocking=True) if isinstance(v, torch.Tensor) else v)
                for k, v in batch.items()} if isinstance(batch, dict) else batch

    # ---- validation ------------------------------------------------------------------------------------------------
    def _val_loader(self, model, val_dataloaders):
        """The validation loader when validation is enabled, else None (`val_dataloader()` is then not called)."""
        if type(model).validation_step is LightningModule.validation_step or self.limit_val_batches == 0:
            return None
        if val_dataloaders is not None:
            return val_dataloaders
        return self.datamodule.val_dataloader() if self.datamodule is not None else None

    @staticmethod
    def _num_batches(loader, limit, name):
        """PL's `_parse_num_batches`: the loader's batch count under an int (count) or float (fraction) limit."""
        try:
            n = len(loader)
        except TypeError:
            n = float("inf")
        if isinstance(limit, int):
            return min(n, limit)
        if n == float("inf"):
            if limit != 1.0:
                raise ValueError(f"{name}={limit} needs a loader with a length")
            return n
        batches = int(n * limit)
        if batches == 0 and limit > 0.0 and n > 0:
            raise ValueError(f"{name}={limit} of {n} batches leaves none; use at least {1.0 / n} or an int")
        return batches

    def _val_check_batch(self, train_loader):
        try:
            n_train = len(train_loader)
        except TypeError:
            n_train = float("inf")
        vci = self.val_check_interval
        if isinstance(vci, int):
            if vci > n_train and self.check_val_every_n_epoch is not None:
                raise ValueError(f"val_check_interval ({vci}) must be less than or equal to the number of the training "
                                 f"batches ({n_train}). To disable validation set limit_val_batches to 0; to validate "
                                 "every N batches across epochs set check_val_every_n_epoch=None.")
            return vci
        if self.check_val_every_n_epoch is None:
            raise ValueError(f"val_check_interval should be an integer when check_val_every_n_epoch=None, found {vci!r}")
        if n_train == float("inf"):
            if vci != 1.0:
                raise ValueError(f"val_check_interval={vci} needs a training loader with a length")
            return n_train       # validate once the epoch has ended
        return max(1, int(n_train * vci))

    def _should_check_val_epoch(self):
        n = self.check_val_every_n_epoch
        return n is None or (self.current_epoch + 1) % n == 0

    @staticmethod
    def _batch_size(batch):
        """PL's `extract_batch_size`: dim 0 of the first tensor found in the batch."""
        if isinstance(batch, torch.Tensor):
            return batch.shape[0] if batch.dim() else 1
        items = batch.values() if isinstance(batch, dict) else batch if isinstance(batch, (list, tuple)) else ()
        for v in items:
            bs = Trainer._batch_size(v)
            if bs is not None:
                return bs
        return None

    def _log_val(self, name, value, sync_dist, device):
        """LightningModule.log inside a validation run: accumulate (v * batch size, batch size) on the device."""
        v = value.detach() if isinstance(value, torch.Tensor) else torch.tensor(float(value))
        v = v.to(device=device, dtype=torch.float64).reshape(())
        bs = self._val_batch_size
        entry = self._val_acc.get(name)
        if entry is None:
            entry = self._val_acc[name] = [torch.zeros(2, dtype=torch.float64, device=device), bool(sync_dist)]
        entry[0][0] += v * bs
        entry[0][1] += bs

    def _run_validation(self, model, loader, n_batches, device, sanity=False):
        rng = (random.getstate(), np.random.get_state(), torch.get_rng_state(),
               torch.cuda.get_rng_state_all() if torch.cuda.is_available() and torch.cuda.is_initialized() else None)
        self.sanity_checking = sanity
        self._val_acc = {}
        model.eval()
        try:
            with torch.no_grad():
                for batch_idx, batch in enumerate(loader):
                    if batch_idx >= n_batches:
                        break
                    self._val_batch_size = self._batch_size(batch) or 1
                    model.validation_step(self._to_device(batch, device), batch_idx)
            acc, self._val_acc = self._val_acc, None
            for sums, sync in acc.values():
                if sync and self.world_size > 1:
                    dist.all_reduce(sums, op=dist.ReduceOp.SUM)
            names = list(acc)
            sums = torch.stack([acc[k][0] for k in names]).tolist() if names else []   # the run's one device->host read
        finally:
            self._val_acc = None
            self.sanity_checking = False
            model.train()
            random.setstate(rng[0]); np.random.set_state(rng[1]); torch.set_rng_state(rng[2])
            if rng[3] is not None:
                torch.cuda.set_rng_state_all(rng[3])
        if sanity:
            return {}
        metrics = {k: s / max(n, 1) for k, (s, n) in zip(names, sums)}
        self._val_names.update(metrics)
        self.callback_metrics.update(metrics)
        if self.logger is not None and self.global_rank == 0 and metrics:
            self.logger.log_metrics(metrics, self.global_step)
        return metrics

    # ---- fit -----------------------------------------------------------------------------------------------------
    def fit(self, model, datamodule=None, ckpt_path=None, train_dataloaders=None, val_dataloaders=None):
        from fsb200.engine import ZeroEngine
        self.lightning_module, self.datamodule = model, datamodule
        model.trainer = self
        if datamodule is not None:
            datamodule.trainer = self
        self._setup_environment()
        if datamodule is not None:
            datamodule.setup("fit")
        if train_dataloaders is not None:
            self._train_loader = train_dataloaders
        model.setup("fit")
        self.optimizers, self.lr_scheduler_configs = self._unpack_optimizers(model.configure_optimizers())
        opt = self.optimizers[0]
        fsb_model = self._find_fsb_model(model)
        tp_group = getattr(fsb_model, "tp_group", None)
        tp = getattr(fsb_model, "tp", 1)
        dp_group = None
        if tp > 1:   # tensor parallelism: ZeRO shards over the data-parallel group (ranks with the same tensor-parallel rank)
            from fengshen.models.megatron import mpu
            dp_group = mpu.get_data_parallel_group()
        if fsb_model.flat.world_size != self.world_size // tp:
            raise RuntimeError(f"model laid out for world_size {fsb_model.flat.world_size}, job has {self.world_size}; "
                               "construct the model inside LightningModule.setup() (as the reference scripts do)")
        g0 = opt.param_groups[0]
        wd = max(g.get("weight_decay", 0.0) for g in opt.param_groups)
        clip = getattr(self.strategy, "gradient_clipping", 0.0) or (self.gradient_clip_val or 0.0)
        betas = g0.get("betas", (0.9, 0.999))
        self.engine = ZeroEngine(fsb_model, lr=g0["lr"], betas=betas, eps=g0.get("eps", 1e-8), weight_decay=wd,
                                 grad_clip=clip, ga_steps=self.accumulate_grad_batches,
                                 stage=getattr(self.strategy, "stage", 2),
                                 overlap_comm=getattr(self.strategy, "overlap_comm", True),
                                 process_group=dp_group, tp_group=tp_group)
        ckpt_path = ckpt_path or self.resume_from_checkpoint
        if ckpt_path:
            self._load_checkpoint(ckpt_path)
            # the loader built for get_total_steps() (model.setup -> trainer._train_dl()) holds a sampler created with
            # consumed_samples = 0; rebuild it now that on_load_checkpoint has restored the counter, as PL does
            if train_dataloaders is None:
                self._train_loader = None
        for cb in self.callbacks:
            cb.on_fit_start(self, model)
        loader = self._train_dl()
        device = fsb_model.flat.params.device
        val_loader = self._val_loader(model, val_dataloaders)
        if val_loader is not None:
            self.val_check_batch = self._val_check_batch(loader)
            n_val = self._num_batches(val_loader, self.limit_val_batches, "limit_val_batches")
            if n_val == 0:       # an empty validation loader: no validation (PL's loop skips itself)
                val_loader = None
        if val_loader is not None:
            n_sanity = n_val if self.num_sanity_val_steps == -1 else min(self.num_sanity_val_steps, n_val)
            if n_sanity > 0:
                self._run_validation(model, val_loader, n_sanity, device, sanity=True)
        total_batch_idx = self.global_step * self.accumulate_grad_batches - 1   # counts across epochs, continues on resume
        done = False
        micro = 0
        while not done:
            stopped_mid_epoch = False
            sampler = getattr(loader, "batch_sampler", None)
            if hasattr(sampler, "set_epoch"):
                sampler.set_epoch(self.current_epoch)
            for batch_idx, batch in enumerate(loader):
                batch = self._to_device(batch, device)
                loss = model.training_step(batch, batch_idx)
                loss = loss["loss"] if isinstance(loss, dict) else loss
                loss.backward()
                self.engine.backward_done()
                micro += 1
                self.just_stepped = False
                if micro % self.accumulate_grad_batches == 0:
                    self.engine.step(lr=opt.param_groups[0]["lr"])
                    opt.step()  # hyper-parameter carrier: a no-op (FusedAdam shim) or grad-less torch optimizer
                    for sc in self.lr_scheduler_configs:
                        if sc.get("interval", "epoch") == "step":
                            sc["scheduler"].step()
                    self.global_step += 1
                    self.fit_loop.epoch_loop._batches_that_stepped += 1
                    self.just_stepped = True
                    if self.logger is not None and self.global_rank == 0 and \
                            self.global_step % max(1, self.log_every_n_steps) == 0:
                        self.logger.log_metrics({k: float(v) for k, v in self.callback_metrics.items()
                                                 if not isinstance(v, str) and k not in self._val_names}, self.global_step)
                for cb in self.callbacks:
                    cb.on_train_batch_end(self, model, loss, batch, batch_idx)
                total_batch_idx += 1
                if val_loader is not None and self._should_check_val_epoch():
                    i = total_batch_idx if self.check_val_every_n_epoch is None else batch_idx
                    if (i + 1) % self.val_check_batch == 0:
                        self._run_validation(model, val_loader, n_val, device)
                if self.max_steps and self.max_steps > 0 and self.global_step >= self.max_steps:
                    done = True
                    stopped_mid_epoch = True
                    break
            if val_loader is not None and self.val_check_batch == float("inf") and not stopped_mid_epoch and \
                    self._should_check_val_epoch():   # a training loader without a length: validate at the epoch's end
                self._run_validation(model, val_loader, n_val, device)
            for sc in self.lr_scheduler_configs:
                if sc.get("interval", "epoch") == "epoch":
                    sc["scheduler"].step()
            for cb in self.callbacks:
                cb.on_train_epoch_end(self, model)
            if not stopped_mid_epoch:   # max_steps hit inside the epoch: it is not complete (a resumed run must reuse its
                self.current_epoch += 1  # permutation seed, universal_sampler.py:104-113)
            if self.max_epochs and self.max_epochs > 0 and self.current_epoch >= self.max_epochs:
                done = True
        self.engine.wait_params()
        for cb in self.callbacks:
            cb.on_fit_end(self, model)
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def predict(self, model, datamodule=None, ckpt_path=None):
        self.lightning_module, self.datamodule = model, datamodule
        model.trainer = self
        if datamodule is not None:
            datamodule.trainer = self
            datamodule.setup("predict")
        self._setup_environment()
        model.setup("predict")
        outs = []
        with torch.no_grad():
            for i, batch in enumerate(datamodule.predict_dataloader() or []):
                outs.append(model.predict_step(batch, i))
        return outs

    # ---- checkpoints: a directory per .ckpt, DeepSpeed layout (SURVEY.md §3.4) --------------------------------------
    def save_checkpoint(self, path, weights_only=False):
        ck = os.path.join(path, "checkpoint")
        if self.global_rank == 0:
            os.makedirs(ck, exist_ok=True)
        if self.world_size > 1:
            dist.barrier()
        module = self.lightning_module
        if self.engine is not None:
            self.engine.wait_params()   # the parameter all-gather of the last step may still be in flight
        tp = getattr(self._find_fsb_model(module), "tp", 1) if module is not None else 1
        consumed = self.global_step * self.accumulate_grad_batches * (self.world_size // max(1, tp)) * \
            int(getattr(getattr(self.datamodule, "hparams", {}), "train_batchsize", 1) or 1)
        if self.global_rank == 0:
            state = {"module": {k: v.detach().cpu() for k, v in module.state_dict().items()},
                     # DeepSpeed's own counters (global_steps / global_samples) next to PL's client state (global_step / epoch):
                     # pretrain_erlangshen.py:192-197 reads checkpoint["global_step"], finetune_ziya_llama.py:180-183 'global_samples'
                     "global_steps": self.global_step, "global_step": self.global_step, "global_samples": consumed,
                     "epoch": self.current_epoch,
                     "lr_schedulers": [sc["scheduler"].state_dict() for sc in self.lr_scheduler_configs]}
            module.on_save_checkpoint(state)
            torch.save(state, os.path.join(ck, "mp_rank_00_model_states.pt"))
        if not weights_only and self.engine is not None:
            sd = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in self.engine.state_dict().items()}
            torch.save(sd, os.path.join(ck, f"zero_pp_rank_{self.global_rank}_mp_rank_00_optim_states.pt"))
        if self.world_size > 1:
            dist.barrier()

    def _load_checkpoint(self, path):
        ck = os.path.join(path, "checkpoint")
        state = torch.load(os.path.join(ck, "mp_rank_00_model_states.pt"), map_location="cpu", weights_only=False)
        module = self.lightning_module
        fsb_model = self._find_fsb_model(module)
        own = module.state_dict()
        with torch.no_grad():
            for k, v in state["module"].items():
                if k in own:
                    own[k].copy_(v.to(own[k].device, own[k].dtype))
        self.global_step = int(state.get("global_steps", 0))
        self.current_epoch = int(state.get("epoch", 0))
        for sc, sd in zip(self.lr_scheduler_configs, state.get("lr_schedulers", [])):
            sc["scheduler"].load_state_dict(sd)
            # LambdaLR.load_state_dict restores the counters but not optimizer.param_groups[*]['lr'], which is what the
            # next engine.step() reads: re-derive it from the restored schedule (otherwise the first resumed step runs at
            # the schedule's step-0 learning rate, 0 under warm-up)
            last = sc["scheduler"].get_last_lr() if hasattr(sc["scheduler"], "get_last_lr") else None
            opt = getattr(sc["scheduler"], "optimizer", None)
            if last is not None and opt is not None:
                for g, lr in zip(opt.param_groups, last):
                    g["lr"] = lr
        opt_path = os.path.join(ck, f"zero_pp_rank_{self.global_rank}_mp_rank_00_optim_states.pt")
        if os.path.exists(opt_path):
            shard = torch.load(opt_path, map_location=fsb_model.flat.params.device, weights_only=False)
            if not isinstance(shard, dict) or shard.get("format") != "fsb200-zero-shard-v1":
                raise RuntimeError(f"{opt_path}: not an fsb200 optimizer shard (format key missing). DeepSpeed's own "
                                   "zero_pp_rank_* payload cannot be resumed by this engine: load the module weights only "
                                   "(delete / move the optimizer shard) or resume with the reference stack.")
            self.engine.load_state_dict(shard)
        else:  # weights-only checkpoint: rebuild the fp32 master copy from the loaded bf16 parameters
            for i in range(len(fsb_model.flat.buckets)):
                self.engine._seg(self.engine.master, i).copy_(fsb_model.flat.bucket_slice(i, self.engine.rank).float())
        module.on_load_checkpoint(state)
