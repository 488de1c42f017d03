"""GPU: dropout through the training stack. The Erlangshen recipe (examples/pretrain_erlangshen_bert.py through fsb200.launch)
on a model directory whose config sets hidden / attention dropout 0.1 — the values the released Erlangshen configs carry —
trains, checkpoints and resumes; and validation inside Trainer.fit (eval mode) draws no masks, so training with a validation run
after every step is bit-identical to training without one."""
import json
import os
import sys

import pytest
import torch

import hf_fixtures as F
import hf_recipes as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "fengshen-lm_b200", "compat")):
    if p not in sys.path:
        sys.path.insert(0, p)
import hf_oracle as H  # noqa: E402  (checker only)


@pytest.fixture
def launched(monkeypatch):
    monkeypatch.syspath_prepend(os.path.join(F.ROOT, "fengshen-lm_b200"))
    saved_path = list(sys.path)
    import fsb200.hf as hf
    import fsb200.launch as launch
    launch.prepare(R.EXAMPLE)
    yield hf
    hf.uninstall()
    sys.path[:] = saved_path


def test_erlangshen_recipe_with_dropout_trains_checkpoints_and_resumes(launched, tmp_path, monkeypatch):
    plain_dir = F.bert_dir

    def dropout_dir(path, **kw):
        cfg = plain_dir(path, **kw)
        cfg.update(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump(cfg, f)
        return cfg

    monkeypatch.setattr(F, "bert_dir", dropout_dir)
    trainer, module = R.erlangshen_recipe(tmp_path, monkeypatch, min_drop=0.3)
    model = module.model
    assert (model.p_hidden, model.p_attn) == (0.1, 0.1) and model.dropout_seed is not None
    # the resumed run trained 16 steps of one micro-batch each: one stream base per forward
    assert int(model.dropout_counter.item()) == 16 * model.dropout_sites


def _batches(n, seed):
    out = []
    for i in range(n):
        b = H.make_mlm_batch(H.BERT_SMALL["vocab_size"], 2, 64, seed=seed + i, nsp=True, pad_tail=5)
        out += [{k: v[j] for k, v in b.items()} for j in range(2)]
    return out


def _fit(tmp, validate, strategy):
    import pytorch_lightning as pl
    from fsb200.models.bert import MegatronBertForPreTraining
    from transformers import MegatronBertConfig

    class Module(pl.LightningModule):
        def setup(self, stage=None):
            torch.manual_seed(0)      # weights and the dropout seed
            cfg = MegatronBertConfig(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.2, hidden_act="gelu_new",
                                     **H.BERT_SMALL)
            self.model = MegatronBertForPreTraining(cfg, device="cuda")
            self.losses, self.val_counters = [], []

        def configure_optimizers(self):
            return torch.optim.AdamW(self.parameters(), lr=1e-3, weight_decay=0.01)

        def training_step(self, b, batch_idx):
            loss = self.model(**b).loss
            self.losses.append(loss.detach().clone())
            return loss

        def validation_step(self, b, batch_idx):
            assert not self.model.training
            self.val_counters.append(int(self.model.dropout_counter.item()))
            self.log("val_loss", self.model(**b).loss)

    train = torch.utils.data.DataLoader(_batches(6, 10), batch_size=2)
    val = torch.utils.data.DataLoader(_batches(2, 90), batch_size=2)
    kw = dict(val_check_interval=1, num_sanity_val_steps=2) if validate else dict(num_sanity_val_steps=0)
    trainer = pl.Trainer(strategy=strategy, max_steps=6, max_epochs=None, default_root_dir=str(tmp), **kw)
    module = Module()
    trainer.fit(module, train_dataloaders=train, val_dataloaders=val if validate else None)
    return trainer, module


@pytest.mark.parametrize("strategy", ["deepspeed_stage_1", "deepspeed_stage_2"])
def test_validation_with_dropout_leaves_training_bit_identical(tmp_path, strategy):
    plain, pm = _fit(tmp_path / "plain", False, strategy)
    trainer, vm = _fit(tmp_path / "val", True, strategy)
    assert trainer.global_step == plain.global_step == 6
    sites = vm.model.dropout_sites
    # sanity runs see the untouched counter, every later run the counter of the steps trained so far
    assert vm.val_counters[:2] == [0, 0] and vm.val_counters[2:] == [s * sites for s in range(1, 7) for _ in range(2)]
    assert int(vm.model.dropout_counter.item()) == int(pm.model.dropout_counter.item()) == 6 * sites
    assert torch.equal(torch.stack(vm.losses), torch.stack(pm.losses))
    assert torch.equal(trainer.engine.flat.params, plain.engine.flat.params)
    for k in ("master", "exp_avg", "exp_avg_sq"):
        assert torch.equal(getattr(trainer.engine, k), getattr(plain.engine, k)), k
