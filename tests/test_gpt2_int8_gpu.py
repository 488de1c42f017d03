"""Int8 / int4 weight-only GPT-2 (`load_in_8bit` / `load_in_4bit`): the W8A16 / W4A16 GEMMs with a bias / gelu_new
epilogue (fsb_gemm_w8a16_bias / fsb_gemm_w4a16_bias) against fp64 and against exact answers, and the quantised GPT-2 against
a bf16 GPT-2 holding the dequantised weights: logits, loss, greedy tokens, graph decode, footprint, loading and refusals."""
import gc
import json
import os

import numpy as np
import pytest
import torch

import int4_ref
import int8_ref
import launch_refs as R
import wq_epilogue_refs as E
from launch_census import Recorder
from fsb200 import lib as L
from fsb200 import ops
from fsb200.models import layers
from fsb200.models.gpt2 import GPT2LMHeadModel

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
V = 512
# (n, k) of the four block projections: c_attn, attn.c_proj, mlp.c_fc, mlp.c_proj
SHAPES = {"110m": [(2304, 768), (768, 768), (3072, 768), (768, 3072)],
          "3.5b": [(9216, 3072), (3072, 3072), (12288, 3072), (3072, 12288)]}
ROWS = (1, 3, 8, 17, 64, 257, 2048)
GEMM = {"int8": ops.gemm_w8a16, "int4": ops.gemm_w4a16}
QUANT = {"int8": ops.quantize_w8, "int4": ops.quantize_w4}
VERIFY = {"int8": E.verify_gemm_w8a16, "int4": E.verify_gemm_w4a16}


def _ws(fmt, m, n, k):
    return int(getattr(L.load(), f"fsb_gemm_{'w8a16' if fmt == 'int8' else 'w4a16'}_workspace_bytes")(m, n, k))


def _dequant(fmt, q, s):
    return (q.float() * s[:, None]).to(BF16) if fmt == "int8" else R.unpack_w4(q, s)


# ------------------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("size", ["110m", "3.5b"])
@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_bias_gemm_matches_fp64(fmt, size):
    g = torch.Generator(device="cuda").manual_seed(1)
    plans = set()
    for n, k in SHAPES[size]:
        w = (torch.randn((n, k), generator=g, device="cuda") * 0.02).to(BF16)
        q, s = QUANT[fmt](w)
        bias = (torch.randn((n,), generator=g, device="cuda") * 0.5).to(BF16)
        for m in ROWS:
            a = torch.randn((m, k), generator=g, device="cuda").to(BF16)
            plans.add(_ws(fmt, m, n, k) > 0)
            for epi in (L.EPI_NONE, L.EPI_GELU_TANH):
                out = GEMM[fmt](a, q, s, bias=bias, epilogue=epi)
                VERIFY[fmt](R.Bound(f"{fmt} {m}x{n}x{k} epi{epi}"), a, q, s, out, bias, epi)
    assert plans == {True, False}, f"{fmt} {size}: the split and the unsplit plan did not both run ({plans})"


def _on_grid(fmt, n, k, g):
    """A bf16 weight [n, k] that quantises exactly (codes on the grid, power-of-two scales, each row / group reaching the
    largest code), its (q, s), and the dequantised weight, which equals it."""
    top = 127 if fmt == "int8" else 7
    codes = torch.randint(-top, top + 1, (n, k), generator=g, device="cuda")
    step = k if fmt == "int8" else 128
    codes[:, ::step] = top                                                      # every row / group reaches the largest code
    exps = torch.randint(-9, -4, (n, 1 if fmt == "int8" else k // 128), generator=g, device="cuda")
    scale = torch.pow(2.0, exps.float()).repeat_interleave(step, 1)
    w = (codes.float() * scale).to(BF16)
    q, s = QUANT[fmt](w)
    deq = _dequant(fmt, q, s)
    assert torch.equal(deq, w), "the grid weight did not survive quantisation exactly"
    return q, s, w


@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_bias_gemm_equals_the_bf16_gemm_on_exact_inputs(fmt):
    """Grid weights, small-integer activations and a coarse bias make every sum exact in fp32, so the _bias GEMM must equal
    fsb_gemm_bf16 NN with the same bias + GELU on the dequantised weight bit for bit, in the split plan as in the unsplit
    one: a bias added once per split, or scale and bias in the wrong order, changes the bits."""
    g = torch.Generator(device="cuda").manual_seed(2)
    plans = set()
    for n, k in [(3072, 3072), (12288, 3072), (3072, 12288), (768, 768)]:
        q, s, w = _on_grid(fmt, n, k, g)
        wt = w.t().contiguous()                                                 # [in, out]: a Conv1D weight
        bias = (torch.randint(-64, 65, (n,), generator=g, device="cuda").float() / 8).to(BF16)
        for m in (1, 5, 64, 2048):
            a = torch.randint(-3, 4, (m, k), generator=g, device="cuda").to(BF16)
            plans.add(_ws(fmt, m, n, k) > 0)
            for epi in (L.EPI_NONE, L.EPI_GELU_TANH):
                got = GEMM[fmt](a, q, s, bias=bias, epilogue=epi)
                want = ops.gemm(L.GEMM_NN, a, wt, bias=bias, epilogue=epi)
                R.Bound(f"{fmt} {m}x{n}x{k} epi{epi}").exact("D against the bf16 GEMM", got, want)
    assert plans == {True, False}, f"{fmt}: the split and the unsplit plan did not both run ({plans})"


@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_bias_gemm_graph_replay_equals_eager(fmt):
    g = torch.Generator(device="cuda").manual_seed(3)
    n, k = 3072, 3072
    q, s = QUANT[fmt]((torch.randn((n, k), generator=g, device="cuda") * 0.02).to(BF16))
    bias = torch.randn((n,), generator=g, device="cuda").to(BF16)
    for m in (1, 8, 300):
        a = torch.randn((m, k), generator=g, device="cuda").to(BF16)
        out = torch.empty((m, n), dtype=BF16, device="cuda")
        eager = GEMM[fmt](a, q, s, bias=bias, epilogue=L.EPI_GELU_TANH)
        GEMM[fmt](a, q, s, out=out, bias=bias, epilogue=L.EPI_GELU_TANH)    # warm-up: workspace and smem attribute
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            GEMM[fmt](a, q, s, out=out, bias=bias, epilogue=L.EPI_GELU_TANH)
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager), (fmt, m)


@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_bias_gemm_refuses_malformed_inputs(fmt):
    name = f"fsb_gemm_{'w8a16' if fmt == 'int8' else 'w4a16'}_bias"
    m, n, k = 4, 256, 256
    q, s = QUANT[fmt]((torch.randn((n, k), device="cuda") * 0.02).to(BF16))
    a = torch.randn((m, k), device="cuda").to(BF16)
    d = torch.empty((m, n), dtype=BF16, device="cuda")
    bias = torch.zeros((n + 8,), dtype=BF16, device="cuda")
    ws = _ws(fmt, m, n, k)
    wsb = torch.empty((max(ws, 16),), dtype=torch.uint8, device="cuda")

    def call(bias_ptr, epi):
        L.call(name, m, n, k, a.data_ptr(), k, q.data_ptr(), s.data_ptr(), bias_ptr, epi, d.data_ptr(), n,
               wsb.data_ptr(), ws, torch.cuda.current_stream().cuda_stream)
    call(bias.data_ptr(), L.EPI_GELU_TANH)                                      # well-formed: accepted
    for bias_ptr, epi, what in ((None, L.EPI_NONE, "NULL"), (bias.data_ptr() + 2, L.EPI_NONE, "aligned"),
                                (bias.data_ptr(), L.EPI_GELU_ERF, "epilogue"), (bias.data_ptr(), 7, "epilogue")):
        with pytest.raises(RuntimeError, match=what):
            call(bias_ptr, epi)
    with pytest.raises(RuntimeError, match="bias"):
        GEMM[fmt](a, q, s, epilogue=L.EPI_GELU_TANH)                           # an epilogue without a bias
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------- model
def _cfg(nh, hn, nl=2, npos=128):
    import transformers
    return transformers.GPT2Config(vocab_size=V, n_positions=npos, n_embd=nh * hn, n_layer=nl, n_head=nh,
                                   bos_token_id=3, eos_token_id=3, resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0,
                                   activation_function="gelu_new")


def _weights(cfg, seed):
    """A bf16 GPT-2 state dict with non-zero biases (HF key names, Conv1D weights [in, out])."""
    m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, seed=seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    with torch.no_grad():
        for k, p in m._p.items():
            if k.endswith("bias"):
                p.normal_(0.0, 0.05, generator=g)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    del m
    return sd


def _dequantised_oracle(qm, sd, cfg):
    """A bf16 GPT-2 holding qm's dequantised Conv1D weights and sd's other parameters."""
    sdq = dict(sd)
    for key, (q, s) in qm._wq_targets().items():
        sdq[key] = _dequant(qm.weight_format, q, s).t().contiguous()
    ref = GPT2LMHeadModel(cfg, device="cuda", world_size=1)
    ref.load_reference_state_dict(sdq)
    return ref


def _flag(fmt):
    return {"load_in_8bit": fmt == "int8", "load_in_4bit": fmt == "int4"}


@pytest.mark.parametrize("hn", [64, 96, 128])
@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_quantised_gpt2_matches_the_dequantised_oracle(fmt, hn):
    nh = 4 if hn != 128 else 2
    cfg = _cfg(nh, hn)
    sd = _weights(cfg, seed=5)
    m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, **_flag(fmt))
    m.load_reference_state_dict(sd)
    assert m.flat.grads is None and m.weight_format == fmt
    # q / s: the numpy quantiser applied to the transposed Conv1D weight
    for key in ("transformer.h.1.attn.c_attn.weight", "transformer.h.0.mlp.c_proj.weight"):
        q, s = m._wq_targets()[key]
        w = sd[key].t().float().cpu().numpy()
        if fmt == "int8":
            qn, sn = int8_ref.quantize(w)
            assert np.array_equal(q.cpu().numpy(), qn) and np.array_equal(s.cpu().numpy(), sn), key
        else:
            qn, sn = int4_ref.quantize(w)
            assert np.array_equal(q.cpu().numpy(), int4_ref.pack(qn)), key
            assert np.array_equal(s.float().cpu().numpy(), sn), key
    ref = _dequantised_oracle(m, sd, cfg)
    B, S = 3, 48
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(4, V, (B, S), generator=g).cuda()
    mask = torch.ones_like(ids)
    mask[1, S - 9:] = 0                                                         # a key mask (right padding)
    seg = torch.cat([torch.zeros(B, 20, dtype=torch.int64), torch.ones(B, S - 20, dtype=torch.int64)], 1).cuda()
    pos = torch.cat([torch.arange(20), torch.arange(S - 20)]).expand(B, S).cuda()
    cases = [dict(input_ids=ids, labels=ids), dict(input_ids=ids, attention_mask=mask, labels=ids),
             dict(input_ids=ids, segment_ids=seg, position_ids=pos, labels=ids)]
    with torch.no_grad():
        for kw in cases:
            got, want = m(**kw, return_logits=True), ref(**kw, return_logits=True)
            tol = 4 * 2.0 ** -8 * float(want.logits.float().abs().max())
            err = float((got.logits.float() - want.logits.float()).abs().max())
            assert err <= tol, (sorted(kw), err, tol)
            assert abs(got.loss.item() - want.loss.item()) < 2e-2, sorted(kw)

    # greedy generate with left padding: wherever the oracle is decisive, its argmax is the generated token
    B, S0, new = 3, 20, 10
    ids = torch.randint(4, V, (B, S0), generator=g)
    mask = torch.ones_like(ids)
    for b in range(1, B):
        ids[b, :4 * b], mask[b, :4 * b] = 0, 0
    seqs = m.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), max_new_tokens=new, pad_token_id=0).cpu()
    checked = 0
    with torch.no_grad():
        for b in range(B):
            real = seqs[b, S0 - int(mask[b].sum()):]
            for t in range(new):
                ctx = real[:len(real) - new + t].cuda()
                lg = ref(input_ids=ctx[None], return_logits=True).logits[0, -1].float()
                top = lg.topk(2).values
                if float(top[0] - top[1]) > 2 * 4 * 2.0 ** -8 * float(lg.abs().max()):
                    assert int(lg.argmax()) == int(real[len(ctx)]), (b, t)
                    checked += 1
    assert checked >= new
    del m, ref
    gc.collect(); torch.cuda.empty_cache()


@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_graph_generate_equals_eager(fmt, monkeypatch):
    cfg = _cfg(4, 96)
    m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, seed=7, **_flag(fmt))
    g = torch.Generator().manual_seed(13)
    ids = torch.randint(4, V, (2, 16), generator=g).cuda()
    mask = torch.ones_like(ids)
    mask[1, :5] = 0
    modes = [dict(max_new_tokens=12), dict(max_new_tokens=12, do_sample=True, top_p=0.9, num_return_sequences=3),
             dict(max_new_tokens=10, num_beams=4)]
    for kw in modes:
        runs = []
        for graph in ("1", "0"):
            monkeypatch.setenv("FSB_GENERATE_GRAPH", graph)
            torch.manual_seed(21)
            runs.append(m.generate(input_ids=ids, attention_mask=mask, pad_token_id=0, **kw).cpu())
        assert torch.equal(runs[0], runs[1]), (fmt, kw)


def test_memory_footprint_orders_int4_int8_bf16():
    cfg = _cfg(4, 64)
    h, inner, nl = 256, 1024, 2
    feet = {}
    for fmt in ("bf16", "int8", "int4"):
        m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, **({} if fmt == "bf16" else _flag(fmt)))
        feet[fmt] = m.get_memory_footprint()
        params = m.flat.params.numel() * 2
        grads = 0 if m.flat.grads is None else m.flat.grads.numel() * m.flat.grads.element_size()
        qs = 0
        for n, k in [(3 * h, h), (h, h), (inner, h), (h, inner)]:
            if fmt == "int8":
                qs += n * k + 4 * n
            elif fmt == "int4":
                qs += n * k // 2 + 2 * n * (k // 128)
        buffers = sum(b.numel() * b.element_size() for b in m.buffers())
        assert feet[fmt] == params + grads + nl * qs + buffers, fmt
        if fmt != "bf16":
            assert grads == 0
        del m
    assert feet["int4"] < feet["int8"] < feet["bf16"]


@pytest.mark.parametrize("sharded", [False, True])
@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_from_pretrained_loads_quantised(fmt, sharded, tmp_path):
    from fsb200 import hf
    cfg = _cfg(4, 64)
    src = hf.GPT2LMHeadModel(cfg, device="cuda", world_size=1, seed=3)
    src.save_pretrained(str(tmp_path))
    sd = {k: v.detach().clone() for k, v in src.state_dict().items()}
    if sharded:   # split the checkpoint into two files with an index, as save_pretrained(max_shard_size=...) writes it
        os.remove(tmp_path / "pytorch_model.bin")
        keys = sorted(sd)
        parts = {"pytorch_model-00001-of-00002.bin": keys[:len(keys) // 2],
                 "pytorch_model-00002-of-00002.bin": keys[len(keys) // 2:]}
        for fn, ks in parts.items():
            torch.save({k: sd[k].cpu() for k in ks}, tmp_path / fn)
        with open(tmp_path / "pytorch_model.bin.index.json", "w") as f:
            json.dump({"weight_map": {k: fn for fn, ks in parts.items() for k in ks}}, f)
    m = hf.GPT2LMHeadModel.from_pretrained(str(tmp_path), device_map="auto", **_flag(fmt))
    assert m.weight_format == fmt
    direct = GPT2LMHeadModel(cfg, device="cuda", world_size=1, **_flag(fmt))
    direct.load_reference_state_dict(sd)
    for a, b in zip(m._wq, direct._wq):
        for key in a:
            assert torch.equal(a[key][0], b[key][0]) and torch.equal(a[key][1], b[key][1]), key
    for k, p in direct._p.items():
        assert torch.equal(m._p[k], p), k
    with pytest.raises(NotImplementedError, match="several devices"):
        hf.GPT2LMHeadModel.from_pretrained(str(tmp_path), device_map={"a": 0, "b": 1}, **_flag(fmt))


@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_quantised_gpt2_refusals(fmt, tmp_path):
    from fsb200 import hf
    flag = f"load_in_{fmt[3:]}bit"
    cfg = _cfg(4, 64)
    m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, **_flag(fmt))
    ids = torch.randint(4, V, (2, 16)).cuda()
    with pytest.raises(NotImplementedError, match=flag):
        m(input_ids=ids, labels=ids)                                            # a training forward
    with pytest.raises(NotImplementedError, match=flag):
        m.save_pretrained(str(tmp_path / "out"))
    with pytest.raises(ValueError, match=flag):
        GPT2LMHeadModel(cfg, device="cuda", world_size=1, fp8=True, **_flag(fmt))
    with pytest.raises(ValueError, match="load_in_8bit and load_in_4bit"):
        GPT2LMHeadModel(cfg, device="cuda", world_size=1, load_in_8bit=True, load_in_4bit=True)
    from fsb200.engine import ZeroEngine
    with pytest.raises(NotImplementedError, match=flag):
        ZeroEngine(m, lr=1e-3)
    if fmt == "int4":
        with pytest.raises(RuntimeError, match="load_in_4bit"):
            GPT2LMHeadModel(_cfg(3, 64), device="cuda", world_size=1, load_in_4bit=True)   # n_embd 192
    # the other HF classes refuse the flag instead of loading a bf16 model
    hf.GPT2LMHeadModel(cfg, device="cuda", world_size=1).save_pretrained(str(tmp_path / "gpt2"))
    for cls in (hf.BertForMaskedLM, hf.MegatronBertForPreTraining, hf.MT5ForConditionalGeneration):
        with pytest.raises(NotImplementedError, match=flag):
            cls.from_pretrained(str(tmp_path / "gpt2"), **{flag: True})


# ------------------------------------------------------------------------------------------------------ launch census
@pytest.mark.parametrize("fmt", ["int8", "int4"])
def test_every_launch_of_quantised_gpt2_generate_against_fp64(fmt, monkeypatch):
    """Every launch of int8 / int4 GPT-2 generate at the benchmark's width with 2 layers, the quantisers included, through
    the launch census (the first call of every signature and every decode-attention call checked against fp64)."""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import bench
    import transformers
    w = bench.workload("gpt2-110m")
    cfg = transformers.GPT2Config(vocab_size=w["vocab_size"], n_positions=w["n_positions"], n_embd=w["n_embd"], n_layer=2,
                                  n_head=w["n_head"], bos_token_id=3, eos_token_id=3, resid_pdrop=0.0, embd_pdrop=0.0,
                                  attn_pdrop=0.0, activation_function="gelu_new")
    monkeypatch.setenv("FSB_GENERATE_GRAPH", "0")
    rec = Recorder(E.CHECKERS, check_all=("attn_decode", "kv_append", "kv_reorder"))
    gen = torch.Generator().manual_seed(7)
    ids = torch.randint(4, 50000, (2, 300), generator=gen).cuda()
    rec.install(monkeypatch)
    for f in ("int8", "int4"):   # the table holds the quantisers bound at import: point it at the recorder's wrappers
        monkeypatch.setitem(layers.WQ, f, (getattr(ops, "quantize_w8" if f == "int8" else "quantize_w4"), layers.WQ[f][1]))
    try:
        torch.cuda.synchronize()
        c0 = L.launch_count
        m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, seed=0, **_flag(fmt))
        m.generate(input_ids=ids, max_new_tokens=8)
        m.generate(input_ids=ids[:1], max_new_tokens=6, num_beams=4)
        torch.cuda.synchronize()
        growth = L.launch_count - c0
    finally:
        monkeypatch.undo()
    assert growth - rec.extra_launches == rec.wrapped_launches, "a kernel was reached without going through fsb200.ops"
    op = "gemm_w8a16" if fmt == "int8" else "gemm_w4a16"
    q = "quantize_w8" if fmt == "int8" else "quantize_w4"
    assert any(k[0] == q for k in rec.checked), f"building the {fmt} model made no {q} call"
    gelu = [k for k in rec.checked if k[0] == op and ("epilogue", L.EPI_GELU_TANH) in k[1]]
    assert gelu, f"no {op} call with the GELU epilogue was checked"
    assert any(k[0] == "kv_reorder" for k in rec.checked), "beam search made no kv_reorder call"
    del m
    gc.collect(); torch.cuda.empty_cache()
