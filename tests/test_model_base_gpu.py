"""GPU: the engine-facing surface every fsb200 model class shares (fsb200/models/base.py). Parameters are views into the flat
bf16 buffer, so the reference scripts' dtype / device calls (`.from_pretrained(..., torch_dtype=torch.half).cuda()`) must leave
them there; and a reference state dict loads only with every parameter present at its shape."""
import re
from types import SimpleNamespace

import pytest
import torch

from fsb200.models.bert import BertForMaskedLM, MegatronBertForPreTraining
from fsb200.models.gpt2 import GPT2LMHeadModel
from fsb200.models.llama import LlamaForCausalLM
from fsb200.models.t5 import MT5ForConditionalGeneration

pytestmark = pytest.mark.gpu

V = 512
_BERT = dict(vocab_size=V, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512,
             max_position_embeddings=128, type_vocab_size=2)
MODELS = {
    "gpt2": (GPT2LMHeadModel, dict(vocab_size=V, n_positions=128, n_embd=256, n_layer=2, n_head=4)),
    "bert": (BertForMaskedLM, _BERT),
    "megatronbert": (MegatronBertForPreTraining, _BERT),
    "mt5": (MT5ForConditionalGeneration, dict(vocab_size=V, d_model=256, d_kv=64, d_ff=512, num_layers=2, num_heads=4,
                                              relative_attention_num_buckets=32, relative_attention_max_distance=128)),
    "llama": (LlamaForCausalLM, dict(vocab_size=V, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                     rms_norm_epsilon=1e-6, max_position_embeddings=2048, rotary_emb_base=10000,
                                     llama_mlp_multiple_of=256)),
}


def _model(name, seed=0):
    cls, cfg = MODELS[name]
    return cls(SimpleNamespace(**cfg), device="cuda", seed=seed)


@torch.no_grad()
def _loss(model):
    ids = torch.randint(1, V, (2, 64), generator=torch.Generator().manual_seed(7))
    return model(input_ids=ids.cuda(), labels=ids.cuda()).loss.item()


@pytest.mark.parametrize("name", list(MODELS))
def test_dtype_and_device_calls_keep_parameters_in_the_flat_buffers(name):
    model = _model(name)
    before = _loss(model)
    for call in (lambda m: m.cuda(), lambda m: m.half(), lambda m: m.bfloat16(), lambda m: m.to(torch.float16),
                 lambda m: m.to("cuda")):
        assert call(model) is model
    params, grads = model.flat.params.untyped_storage().data_ptr(), model.flat.grads.untyped_storage().data_ptr()
    for n, p in model.named_parameters():
        assert (p.dtype, p.untyped_storage().data_ptr()) == (torch.bfloat16, params), n
        assert p.main_grad.untyped_storage().data_ptr() == grads, n
    assert _loss(model) == before


@pytest.mark.parametrize("name", list(MODELS))
def test_load_reference_state_dict_requires_every_parameter_at_its_shape(name):
    model = _model(name)
    sd = {k: v.float().cpu() for k, v in model.state_dict().items()}
    names = [n for n, _ in model.named_parameters()]
    key = names[len(names) // 2]
    with pytest.raises(KeyError, match=re.escape(key)):
        _model(name).load_reference_state_dict({k: v for k, v in sd.items() if k != key})
    with pytest.raises(ValueError, match=re.escape(key)):
        _model(name).load_reference_state_dict({**sd, key: sd[key][..., :1]})
    other = _model(name, seed=1)
    other.load_reference_state_dict({**sd, "not.a.parameter": torch.zeros(3)})
    assert torch.equal(other.flat.params, model.flat.params)
