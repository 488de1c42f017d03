"""HF-style export / import for the fsb200 model classes (SURVEY.md §8f rank 2): the reference's scripts end a run with
`self.model.save_pretrained(path)` (examples/pretrain_t5/pretrain_t5.py:105-112, examples/pretrain_erlangshen_bert/
pretrain_erlangshen.py on_save_checkpoint) and start the next one with `from_pretrained(path)`. Every fsb200 model keeps the
state-dict key names of the class it stands in for, so the directory written here (config.json + pytorch_model.bin) is read back
by `transformers.<Class>.from_pretrained` as well as by `from_pretrained` below."""
import json
import os

import torch


def _config_dict(cfg):
    if hasattr(cfg, "to_dict"):
        d = cfg.to_dict()
    else:
        d = {k: v for k, v in vars(cfg).items() if not k.startswith("_")}
    return {k: v for k, v in d.items() if isinstance(v, (int, float, str, bool, list, dict, type(None)))}


def wait_params(model):
    """Join the parameter all-gather the engine driving `model` (if any) may still have in flight, before the parameters are
    read from the host."""
    eng = getattr(getattr(model, "param_hook", None), "__self__", None)
    if eng is not None and hasattr(eng, "wait_params"):
        eng.wait_params()


def save_pretrained(model, path, extra_config=None):
    """config.json + pytorch_model.bin (bf16 tensors, HF key names). Waits for an in-flight parameter all-gather first."""
    wait_params(model)
    os.makedirs(path, exist_ok=True)
    cfg = _config_dict(model.config)
    cfg.update(extra_config or {})
    cfg.setdefault("torch_dtype", "bfloat16")
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f, indent=1)
    torch.save({k: v.detach().cpu().clone() for k, v in model.state_dict().items()}, os.path.join(path, "pytorch_model.bin"))


def from_pretrained(model_cls, path, config_cls=None, **model_kwargs):
    """Build `model_cls` from `path/config.json` (through `config_cls(**json)` when given, else a plain namespace) and load
    `path/pytorch_model.bin` (or the shards named by pytorch_model.bin.index.json) with `load_reference_state_dict`."""
    from types import SimpleNamespace
    with open(os.path.join(path, "config.json")) as f:
        raw = json.load(f)
    for k in ("torch_dtype", "dtype", "architectures", "transformers_version"):
        raw.pop(k, None)
    cfg = config_cls(**raw) if config_cls is not None else SimpleNamespace(**raw)
    model = model_cls(cfg, **model_kwargs)
    files = [os.path.join(path, "pytorch_model.bin")]
    idx = os.path.join(path, "pytorch_model.bin.index.json")
    if os.path.exists(idx):
        with open(idx) as f:
            files = sorted({os.path.join(path, v) for v in json.load(f)["weight_map"].values()})
    sd = {}
    for fn in files:
        sd.update(torch.load(fn, map_location="cpu", weights_only=True))
    model.load_reference_state_dict(sd)
    return model
