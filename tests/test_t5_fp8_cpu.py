"""CPU checks for FP8 training of mT5: the shared-input path of Fp8Linear (the encoder output quantised once for every
decoder layer's cross k|v projection) on recording stand-ins for the two FP8 ops, and `from_pretrained(path, fp8=True)`
reaching the model's constructor."""
import inspect

import pytest
import torch

BF16 = torch.bfloat16


@pytest.fixture
def fake_fp8(monkeypatch):
    """ops.fp8_quantize / ops.gemm_fp8 replaced by stand-ins that record what they were given."""
    from fsb200 import ops
    calls = []

    def quantize(x, fmt, rowwise=True, colwise=False):
        calls.append(("quantize", x, fmt, rowwise, colwise))
        return (x if rowwise else None), (x.t() if colwise else None), torch.ones(1)

    def gemm(a, sa, b, sb, out=None, accumulate=False, **kw):
        calls.append(("gemm", a, b, out, accumulate))
        return torch.zeros(a.shape[0], b.shape[0], dtype=BF16) if out is None else out
    monkeypatch.setattr(ops, "fp8_quantize", quantize)
    monkeypatch.setattr(ops, "gemm_fp8", gemm)
    return calls


def _lin(n=32, k=16):
    from fsb200.models.layers import Fp8Linear, Linear
    w = torch.zeros(n, k, dtype=BF16)
    return Fp8Linear(Linear(w, torch.zeros_like(w)))


def test_shared_codes_are_quantised_once(fake_fp8):
    from fsb200.models.layers import Fp8Linear
    x = torch.zeros(48, 16, dtype=BF16)
    codes = Fp8Linear.quantize_input(x, True)
    assert [c[0] for c in fake_fp8] == ["quantize"] and fake_fp8[0][2:] == ("e4m3", True, True)
    fake_fp8.clear()
    layers = [_lin(), _lin()]
    for lin in layers:
        lin.forward(x, False, codes=codes)
    # each layer casts only its weight, and its GEMM reads the shared row-major codes
    quants = [c for c in fake_fp8 if c[0] == "quantize"]
    gemms = [c for c in fake_fp8 if c[0] == "gemm"]
    assert len(quants) == 2 and all(q[1] is lin.lin.weight for q, lin in zip(quants, layers))
    assert len(gemms) == 2 and all(g[1] is codes[0] for g in gemms)


def test_shared_codes_feed_the_weight_gradient(fake_fp8):
    """What the backward of each cross k|v projection reads of the encoder output is the shared transposed codes and
    scale, and its data gradient accumulates into the caller's buffer after the first layer."""
    from fsb200.models.layers import Fp8Linear
    x = torch.zeros(48, 16, dtype=BF16)
    codes = Fp8Linear.quantize_input(x, True)
    dx = torch.zeros(48, 16, dtype=BF16)
    for i, lin in enumerate((_lin(), _lin())):
        fake_fp8.clear()
        lin.backward(torch.zeros(48, 32, dtype=BF16), codes[1:], False, dx=dx, dx_accumulate=i > 0)
        dgrad, wgrad = [c for c in fake_fp8 if c[0] == "gemm"]
        assert dgrad[3] is dx and dgrad[4] is (i > 0)
        assert wgrad[2] is codes[1] and wgrad[3] is lin.lin.weight_grad


def test_model_and_from_pretrained_take_fp8(tmp_path, monkeypatch):
    """from_pretrained(path, fp8=True) hands fp8 to the model's constructor (stopped there: the model needs CUDA)."""
    import json
    from fsb200 import hf
    from fsb200.models.t5 import MT5ForConditionalGeneration
    assert inspect.signature(MT5ForConditionalGeneration.__init__).parameters["fp8"].default is False
    (tmp_path / "config.json").write_text(json.dumps(dict(vocab_size=512, d_model=256, d_kv=64, d_ff=512, num_layers=2,
                                                          num_heads=4, feed_forward_proj="gated-gelu")))
    (tmp_path / "pytorch_model.bin").write_bytes(b"")
    seen = []

    class Stop(Exception):
        pass

    def init(self, config, *args, **kwargs):
        seen.append(kwargs)
        raise Stop
    monkeypatch.setattr(MT5ForConditionalGeneration, "__init__", init)
    for kw in (dict(fp8=True), {}):
        with pytest.raises(Stop):
            hf.MT5ForConditionalGeneration.from_pretrained(str(tmp_path), **kw)
    assert seen[0].get("fp8") is True and "fp8" not in seen[1]
