"""`fengshen.models.llama.modeling_llama.LlamaForCausalLM` -> fsb200.models.llama.LlamaForCausalLM, plus the
`from_pretrained(path, torch_dtype=...)` entry the scripts use (examples/ziya_llama/finetune_ziya_llama.py:102-107)."""
import json
import os

import torch

from fsb200.models.export import wait_params
from fsb200.models.llama import LlamaForCausalLM as _FsbLlama
from .configuration_llama import LlamaConfig


class LlamaForCausalLM(_FsbLlama):
    config_class = LlamaConfig

    def __init__(self, config, **kw):
        for k, want in (("rotary_pct", 1), ("pos_emb", "rotary"), ("norm", "rmsnorm"), ("mlp_type", "llama"),
                        ("hidden_dropout", 0), ("attention_dropout", 0), ("use_bias_in_attn_linear", False)):
            have = getattr(config, k, want)
            if have != want:
                raise NotImplementedError(f"fsb200 LlamaForCausalLM: config.{k}={have!r} is outside the Ziya-LLaMA "
                                          f"hot path (only {want!r} is implemented)")
        if "tp_group" not in kw:   # built inside LightningModule.setup(), after the strategy initialised mpu (as the reference)
            from fengshen.models.megatron import mpu
            if mpu.get_model_parallel_world_size() > 1:
                kw["tp_group"] = mpu.get_model_parallel_group()
        super().__init__(config, **kw)

    @classmethod
    def from_pretrained(cls, path, torch_dtype=None, load_in_8bit=False, device_map=None, load_in_4bit=False, **kw):
        """Loads config.json + pytorch_model.bin (or the sharded index) written by the reference's save_pretrained /
        hf_to_fs.py. torch_dtype is accepted for signature parity; parameters are stored in bf16.

        load_in_8bit=True (examples/ziya_inference/hf_quantizatin_inference.py:20-22): an inference-only model whose layer
        projections are int8 (fsb200/models/llama.py). The checkpoint is read one shard file at a time and each shard's
        matrices are quantised on the device before the next file is read, so host memory holds one shard. HF-format
        directories are converted first with `fengshen.utils.llama_convert.hf_to_fs_state_dict`.
        load_in_4bit=True (hf_quantizatin_inference.py:3,16): the same with int4 projections (one bf16 scale per row and
        group of 128 k), loaded the same way. Passing both flags raises ValueError.
        fp8=True (passed on to the model like the other keywords): train the layer projections in FP8 (fsb200/models/llama.py).
        gradient_checkpointing=True (passed on the same way): recompute each layer in the backward instead of keeping its
        activations, as `model.gradient_checkpointing_enable()` does after loading.
        device_map: None, "auto" or one device (the model lives on one GPU); a map over several devices raises."""
        if device_map is not None and device_map != "auto":
            if isinstance(device_map, dict):
                devs = {torch.device(f"cuda:{v}" if isinstance(v, int) else v) for v in device_map.values()}
                if len(devs) != 1:
                    raise NotImplementedError(f"fsb200 LlamaForCausalLM: device_map over several devices {sorted(map(str, devs))}"
                                              " is not implemented; the model runs on one GPU")
                device_map = next(iter(devs))
            dev = torch.device(f"cuda:{device_map}" if isinstance(device_map, int) else device_map)
            kw.setdefault("device", dev)
        with open(os.path.join(path, "config.json")) as f:
            raw = json.load(f)
        raw.pop("torch_dtype", None); raw.pop("architectures", None); raw.pop("model_type", None)
        model = cls(LlamaConfig(**raw), load_in_8bit=load_in_8bit, load_in_4bit=load_in_4bit, **kw)
        idx = os.path.join(path, "pytorch_model.bin.index.json")
        files = [os.path.join(path, "pytorch_model.bin")]
        if os.path.exists(idx):
            with open(idx) as f:
                files = sorted({os.path.join(path, v) for v in json.load(f)["weight_map"].values()})
        if model.weight_format != "bf16":
            loaded, missing = set(), None
            for fn in files:
                shard = torch.load(fn, map_location="cpu", weights_only=True)
                missing = model._load_quantized_shard(shard, loaded)
                del shard
            if missing:
                raise KeyError(f"missing key in checkpoint {path}: {sorted(missing)[0]}")
            return model
        sd = {}
        for fn in files:
            sd.update(torch.load(fn, map_location="cpu", weights_only=True))
        model.load_reference_state_dict(sd)
        return model

    def save_pretrained(self, path, **_):
        """HF-style export (what the scripts call after training, e.g. examples/pretrain_t5/pretrain_t5.py:105-112 for its
        model): config.json + pytorch_model.bin in the reference's key layout; `from_pretrained(path)` reads it back, and
        `fengshen.utils.llama_convert.fs_to_hf_state_dict` turns it into a transformers LLaMA checkpoint."""
        if self.weight_format != "bf16":
            return super().save_pretrained(path)   # raises: int8 / int4 export is not implemented
        from fengshen.utils.llama_convert import save_pretrained_fs
        wait_params(self)
        cfg = self.config.to_dict() if hasattr(self.config, "to_dict") else vars(self.config)
        save_pretrained_fs({k: v for k, v in self.state_dict().items()}, cfg, path)
