"""CPU checks for FP8 training of GPT-2: which codes and layouts Fp8Conv1D hands to which FP8 GEMM, on recording stand-ins for
the FP8 ops (a gemm_fp8 call with store_transposed=True is recorded as "gemm_fp8_t"), and `from_pretrained(path, fp8=True)`
reaching the model's constructor."""
import inspect

import pytest
import torch

BF16 = torch.bfloat16


@pytest.fixture
def fake_fp8(monkeypatch):
    """ops.fp8_quantize / gemm_fp8 / colsum replaced by stand-ins that record what they were given. A stand-in's
    transposed codes are x.t(), so a layout is recognisable by its shape and strides."""
    from fsb200 import ops
    calls = []

    def quantize(x, fmt, rowwise=True, colwise=False):
        calls.append(("quantize", x, fmt, rowwise, colwise))
        return (x if rowwise else None), (x.t() if colwise else None), torch.ones(1)

    def gemm(a, sa, b, sb, out=None, accumulate=False, store_transposed=False, **kw):
        op = "gemm_fp8_t" if store_transposed else "gemm_fp8"
        calls.append((op, a, b, out, accumulate, kw))
        shape = (b.shape[0], a.shape[0]) if store_transposed else (a.shape[0], b.shape[0])
        return torch.zeros(shape, dtype=BF16) if out is None else out
    monkeypatch.setattr(ops, "fp8_quantize", quantize)
    monkeypatch.setattr(ops, "gemm_fp8", gemm)
    monkeypatch.setattr(ops, "colsum", lambda x, out, accumulate=False: calls.append(("colsum", x, out, accumulate)))
    return calls


def _conv(din=16, dout=48, bias=True):
    from fsb200.models.layers import Fp8Conv1D, Linear
    w = torch.zeros(din, dout, dtype=BF16)
    b = torch.zeros(dout, dtype=BF16) if bias else None
    return Fp8Conv1D(Linear(w, torch.zeros_like(w), b, None if b is None else torch.zeros_like(b), conv1d=True))


def _same(t, ref):
    return t.data_ptr() == ref.data_ptr() and t.shape == ref.shape and t.stride() == ref.stride()


def test_forward_reads_x_row_major_and_the_weights_transposed_codes(fake_fp8):
    from fsb200 import lib as L
    conv = _conv()
    x = torch.zeros(32, 16, dtype=BF16)
    aux = torch.zeros(32, 48, dtype=BF16)
    y, saved = conv.forward(x, True, L.EPI_GELU_TANH, aux)
    (q_x, q_w, g) = fake_fp8
    assert q_x[1] is x and q_x[2:] == ("e4m3", True, True)                   # x: both layouts when saving
    assert q_w[1] is conv.lin.weight and q_w[2:] == ("e4m3", False, True)     # W [in, out]: its transposed codes only
    assert g[0] == "gemm_fp8" and g[1] is x and _same(g[2], conv.lin.weight.t())
    assert g[5] == dict(bias=conv.lin.bias, epilogue=L.EPI_GELU_TANH, aux=aux)
    assert y.shape == (32, 48) and _same(saved[0], x.t())
    fake_fp8.clear()
    _, saved = _conv(bias=False).forward(x, False)
    assert saved is None and fake_fp8[0][2:] == ("e4m3", True, False) and fake_fp8[-1][5] == {}   # plain call


def test_backward_layouts_and_the_transposed_store(fake_fp8):
    conv = _conv()
    x, dy = torch.zeros(32, 16, dtype=BF16), torch.zeros(32, 48, dtype=BF16)
    saved = (x.t(), torch.ones(1))
    dx_buf = torch.zeros(32, 16, dtype=BF16)
    dx = conv.backward(dy, saved, True, dx=dx_buf, dx_accumulate=True)
    q_dy, q_w, dgrad, wgrad, cs = fake_fp8
    assert q_dy[1] is dy and q_dy[2:] == ("e5m2", True, True)
    assert q_w[1] is conv.lin.weight and q_w[2:] == ("e4m3", True, False)    # W [in, out] row-major: dx = dy W^T
    assert dgrad[0] == "gemm_fp8" and dgrad[1] is dy and dgrad[2] is conv.lin.weight
    assert dgrad[3] is dx_buf and dgrad[4] is True and dx is dx_buf
    # dW [in, out] = (dy^T x)^T: A = dy^T codes [out, tokens], B = x^T codes [in, tokens], stored transposed
    assert wgrad[0] == "gemm_fp8_t" and _same(wgrad[1], dy.t()) and wgrad[2] is saved[0]
    assert wgrad[3] is conv.lin.weight_grad and wgrad[4] is True
    assert cs[0] == "colsum" and cs[1] is dy and cs[2] is conv.lin.bias_grad
    fake_fp8.clear()
    conv.backward(dy, saved, False, colsum=False)
    assert [c[0] for c in fake_fp8] == ["quantize", "quantize", "gemm_fp8", "gemm_fp8_t"]
    assert fake_fp8[-1][4] is False


def test_saved_input_is_what_forward_keeps(fake_fp8):
    conv = _conv()
    x = torch.zeros(32, 16, dtype=BF16)
    xt, _ = conv.saved_input(x)
    assert fake_fp8[0][1] is x and fake_fp8[0][2:] == ("e4m3", False, True) and _same(xt, x.t())


def test_layer_types_refuse_the_other_weight_layout():
    from fsb200.models.layers import Fp8Conv1D, Fp8Linear, Linear
    w = torch.zeros(16, 48, dtype=BF16)
    with pytest.raises(ValueError, match="Fp8Conv1D: only \\[in, out\\] Conv1D"):
        Fp8Conv1D(Linear(w, torch.zeros_like(w)))
    with pytest.raises(ValueError, match="Conv1D weight is \\[in, out\\]"):
        Fp8Linear(Linear(w, torch.zeros_like(w), conv1d=True))


def test_model_and_from_pretrained_take_fp8(tmp_path, monkeypatch):
    """from_pretrained(path, fp8=True) hands fp8 to the model's constructor (stopped there: the model needs CUDA)."""
    import json
    from fsb200 import hf
    from fsb200.models.gpt2 import GPT2LMHeadModel
    assert inspect.signature(GPT2LMHeadModel.__init__).parameters["fp8"].default is False
    (tmp_path / "config.json").write_text(json.dumps(dict(model_type="gpt2", vocab_size=512, n_positions=128, n_embd=3072,
                                                          n_layer=1, n_head=32)))
    (tmp_path / "pytorch_model.bin").write_bytes(b"")
    seen = []

    class Stop(Exception):
        pass

    def init(self, config, *args, **kwargs):
        seen.append(kwargs)
        raise Stop
    monkeypatch.setattr(GPT2LMHeadModel, "__init__", init)
    for kw in (dict(fp8=True), {}):
        with pytest.raises(Stop):
            hf.GPT2LMHeadModel.from_pretrained(str(tmp_path), **kw)
    assert seen[0].get("fp8") is True and "fp8" not in seen[1]
