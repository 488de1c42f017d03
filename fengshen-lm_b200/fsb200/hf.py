"""The `transformers` class names the reference's HF-backed recipes instantiate, backed by fsb200 models (SURVEY §8a row A16):

    transformers.GPT2LMHeadModel              fengshen/examples/wenzhong_qa/finetune_wenzhong.py:9,56          (C2)
    transformers.BertForMaskedLM              fengshen/examples/pretrain_bert/pretrain_bert.py:2-8,135-137      (C1)
    transformers.MegatronBertForPreTraining   fengshen/examples/pretrain_erlangshen_bert/pretrain_erlangshen.py:2-6,138-141 (C3)
    transformers.MT5ForConditionalGeneration  fengshen/examples/pretrain_t5/pretrain_t5.py:11,57-59             (C5)

Each keeps the call surface those scripts use — `Class(config)`, `Class.from_pretrained(dir)`, `model(**batch)` returning an
object with `.loss` and `.logits` / `.prediction_logits`, `state_dict()` in HF key names, `save_pretrained(dir)` — and runs the
step on libfsb200.so. `install()` rebinds the four names on the `transformers` module so that an UNMODIFIED script's
`from transformers import MegatronBertForPreTraining` picks them up; `python -m fsb200.launch script.py ...` does that and then
runs the script. GPT2LMHeadModel and MT5ForConditionalGeneration also carry `generate` (KV-cache decoding on the split-KV decode
kernel, HF GenerationMixin semantics: fsb200/generation.py). All four classes apply the config's dropout in training mode
(fsb200/models/gpt2.py, fsb200/models/bert.py, fsb200/models/t5.py). Anything outside the hot path (GPT-2 / mT5 `generate` in
training mode with dropout > 0, generation for the encoder-only BERT classes, output_attentions, generation keywords
fsb200/generation.py does not implement) raises instead of silently differing."""
import json
import os

from .models import bert as _bert
from .models import gpt2 as _gpt2
from .models import t5 as _t5
from .models.export import from_pretrained as _load_dir

_NAMES = ("GPT2LMHeadModel", "BertForMaskedLM", "MegatronBertForPreTraining", "MT5ForConditionalGeneration")
_originals = {}


def _hf_config(name):
    import transformers
    return getattr(transformers, name)


def _device_of_map(device_map, model):
    """The one device a `device_map` (None, "auto", a device, or a dict of devices) places the model on; None for the default
    device. A map over several devices raises: the model runs on one GPU."""
    import torch
    if device_map is None or device_map == "auto":
        return None
    if isinstance(device_map, dict):
        devs = {torch.device(f"cuda:{v}" if isinstance(v, int) else v) for v in device_map.values()}
        if len(devs) != 1:
            raise NotImplementedError(f"fsb200 {model}: device_map over several devices {sorted(map(str, devs))} is not "
                                      "implemented; the model runs on one GPU")
        device_map = next(iter(devs))
    return torch.device(f"cuda:{device_map}" if isinstance(device_map, int) else device_map)


class _HFSurface:
    """from_pretrained / forward defaults shared by the four classes."""
    config_name = None
    RETURN_LOGITS = True     # HF outputs always carry logits; scripts that never read them may set this False to skip a copy
    QUANTIZED = False        # from_pretrained(load_in_8bit / load_in_4bit=True) builds an int8 / int4 model (GPT-2 only)

    def __init__(self, config, *args, **kwargs):
        """The reference's HF-backed scripts build the model in LightningModule.__init__, BEFORE the Trainer has initialised
        torch.distributed (pretrain_erlangshen.py:138-141): take the ZeRO layout from the launcher's environment then."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            kwargs.setdefault("world_size", int(os.environ.get("WORLD_SIZE", "1")))
            if "LOCAL_RANK" in os.environ:
                kwargs.setdefault("device", f"cuda:{int(os.environ['LOCAL_RANK'])}")
        super().__init__(config, *args, **kwargs)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, *model_args, config=None, state_dict=None, **kwargs):
        path = str(pretrained_model_name_or_path)
        if not os.path.isdir(path):
            raise FileNotFoundError(f"fsb200 {cls.__name__}.from_pretrained: {path!r} is not a local directory "
                                    "(there is no hub access on the product path)")
        # model keywords: fp8 exists on BertForMaskedLM, MegatronBertForPreTraining (fsb200/models/bert.py),
        # MT5ForConditionalGeneration (fsb200/models/t5.py) and GPT2LMHeadModel (fsb200/models/gpt2.py); load_in_8bit /
        # load_in_4bit on GPT2LMHeadModel only (the others refuse them rather than load a bf16 model)
        kw = {k: kwargs[k] for k in ("device", "world_size", "seed", "fp8") if k in kwargs}
        for flag in ("load_in_8bit", "load_in_4bit"):
            if kwargs.get(flag):
                if not cls.QUANTIZED:
                    raise NotImplementedError(f"fsb200 {cls.__name__}.from_pretrained: {flag}=True is not implemented for "
                                              "this model (int8 / int4 inference covers GPT2LMHeadModel and LLaMA)")
                kw[flag] = True
        dev = _device_of_map(kwargs.get("device_map"), cls.__name__)
        if dev is not None:
            kw.setdefault("device", dev)
        cfg_cls = _hf_config(cls.config_name)
        if config is not None or state_dict is not None:
            # pretrain_t5.py:34-50: an edited config plus an edited state dict on top of the directory
            if config is None:
                config = cfg_cls.from_pretrained(path)
            model = cls(config, **kw)
            if state_dict is None:
                import torch
                state_dict = torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu", weights_only=True)
            model.load_reference_state_dict(state_dict)
            return model
        with open(os.path.join(path, "config.json")) as f:
            raw = json.load(f)
        for k in ("torch_dtype", "dtype", "architectures", "transformers_version", "model_type"):
            raw.pop(k, None)
        if not (os.path.exists(os.path.join(path, "pytorch_model.bin")) or
                os.path.exists(os.path.join(path, "pytorch_model.bin.index.json"))):
            raise FileNotFoundError(f"fsb200 {cls.__name__}.from_pretrained: no pytorch_model.bin under {path!r} "
                                    "(safetensors checkpoints: convert with transformers' save_pretrained(safe_serialization=False))")
        return _load_dir(cls, path, config_cls=cfg_cls, **kw)

    def forward(self, *args, **kwargs):
        if args:
            raise TypeError(f"fsb200 {type(self).__name__}: pass inputs by keyword (input_ids=..., labels=...), as the "
                            "reference's training_step does")
        for k in ("output_attentions", "output_hidden_states", "past_key_values", "inputs_embeds", "head_mask"):
            if kwargs.get(k) not in (None, False):
                raise NotImplementedError(f"fsb200 {type(self).__name__}: {k} is outside the pretraining hot path")
        kwargs.setdefault("return_logits", self.RETURN_LOGITS)
        return super().forward(**kwargs)


class GPT2LMHeadModel(_HFSurface, _gpt2.GPT2LMHeadModel):
    config_name = "GPT2Config"
    QUANTIZED = True


class BertForMaskedLM(_HFSurface, _bert.BertForMaskedLM):
    config_name = "BertConfig"


class MegatronBertForPreTraining(_HFSurface, _bert.MegatronBertForPreTraining):
    config_name = "MegatronBertConfig"


class MT5ForConditionalGeneration(_HFSurface, _t5.MT5ForConditionalGeneration):
    config_name = "MT5Config"


def _transformers_modules():
    """transformers 5.x re-creates its lazy top-level module on the first heavy attribute access (sys.modules['transformers']
    is a different object afterwards), so: force that access, then patch every module object that can still be reached."""
    import sys
    import transformers as first
    for n in _NAMES:
        getattr(first, n)
    mods = [sys.modules["transformers"]]
    if first is not mods[0]:
        mods.append(first)
    return mods


def install():
    """Rebind the four class names on the `transformers` module (idempotent). Call before the script's own imports run."""
    g = globals()
    for mod in _transformers_modules():
        for n in _NAMES:
            cur = getattr(mod, n)
            if cur is not g[n]:
                _originals.setdefault(n, cur)
                setattr(mod, n, g[n])
        if not hasattr(mod, "MT5Tokenizer"):   # removed in transformers 5.x, where it was `MT5Tokenizer = T5Tokenizer`;
            mod.MT5Tokenizer = mod.T5Tokenizer   # pretrain_t5.py:9 imports it by that name


def uninstall():
    for mod in _transformers_modules():
        for n, c in _originals.items():
            setattr(mod, n, c)
    _originals.clear()
