"""GPU: int4 weight-only LLaMA inference. The quantiser (fsb_quantize_w4) against the numpy restatement of its format in
tests/int4_ref.py, bit for bit (scales and packed bytes); the W4A16 GEMM (fsb_gemm_w4a16) against fp64 over the dequantised
weight W^ = bf16(q * s) with the error bound its fp32 accumulation allows, NaN sentinels, determinism and graph capture;
the `load_in_4bit` LLaMA against the CPU oracle with every projection replaced by W^; graphed against eager generate;
shard-by-shard loading and its memory; and the paths an int4 model refuses."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import int4_ref as R  # noqa: E402
import llama_oracle as O  # noqa: E402
from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402

V = 512
PROJ = ("attention.query_key_value.weight", "attention.dense.weight", "mlp.w1.weight", "mlp.w3.weight", "mlp.w2.weight")


def _bits(s):
    """bf16 tensor -> uint16 numpy bit patterns."""
    return s.cpu().view(torch.int16).numpy().view(np.uint16)


def _ref_bits(s):
    """float32 numpy holding bf16 values -> uint16 bit patterns."""
    return (np.ascontiguousarray(s, dtype=np.float32).view(np.uint32) >> 16).astype(np.uint16)


def _check_quantized(q, s, w):
    """q / s from the library are bit-identical to the numpy restatement applied to w (float32 of the bf16 weight)."""
    qn, sn = R.quantize(w)
    assert np.array_equal(_bits(s), _ref_bits(sn))
    assert np.array_equal(q.cpu().numpy(), R.pack(qn))


# ---- quantiser ---------------------------------------------------------------------------------------------------------
def test_quantize_w4_matches_numpy_bit_for_bit():
    g = torch.Generator().manual_seed(0)
    k = 1024
    rows = [torch.randn(k, generator=g) * 2.0 ** e for e in (-60, -30, -10, 0, 10, 30, 60)]
    gz = torch.randn(k, generator=g)
    gz[256:384] = 0.0
    rows.append(gz)                                                        # an all-zero group inside a non-zero row
    out = torch.randn(k, generator=g) * 1e-2
    out[torch.arange(8) * 128 + torch.arange(8) * 13] = torch.tensor([900.0, -37.0, 5.0, -2e4, 0.3, 77.0, -1e-1, 3e5])
    rows.append(out)                                                       # one outlier per group
    half = torch.zeros(k)                                                  # absmax 7 -> s = 1: exact half-steps
    half[:11] = torch.tensor([7.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 6.5, -6.5, 3.5, -3.5])
    rows.append(half)
    clamp = torch.zeros(k)                                                 # s = bf16(7.0625 / 7) < 7.0625 / 7
    clamp[:3] = torch.tensor([7.0625, -7.0625, 3.5])
    rows.append(clamp)
    rows.append(torch.zeros(k))
    while len(rows) % 8:
        rows.append(torch.randn(k, generator=g))
    w = torch.stack(rows).to(torch.bfloat16)
    wide = torch.full((w.shape[0], k + 72), float("nan"), dtype=torch.bfloat16)
    wide[:, :k] = w
    wn = w.float().numpy()
    for src in (w.cuda(), wide.cuda()[:, :k]):                            # contiguous and strided (ldw > k)
        q, s = ops.quantize_w4(src)
        torch.cuda.synchronize()
        _check_quantized(q, s, wn)
    qn = R.unpack(q.cpu().numpy())
    assert qn[9, :11].tolist() == [7, 0, 2, 2, 0, -2, -2, 6, -6, 4, -4]   # ties to even
    assert qn[10, :3].tolist() == [7, -7, 3]                               # clamp after the scale is rounded
    assert float(s[10, 0]) == 1.0078125
    assert not s[7, 2].item() and not qn[7, 256:384].any() and s[7, 1].item() and s[7, 3].item()
    assert not s[11].any() and not qn[11].any()


def test_quantize_w4_rejects_malformed_inputs():
    with pytest.raises(RuntimeError, match="128"):
        ops.quantize_w4(torch.zeros((256, 520), dtype=torch.bfloat16, device="cuda"))
    w = torch.zeros((256, 640), dtype=torch.bfloat16, device="cuda")
    q = torch.empty((128, 640), dtype=torch.uint8, device="cuda")
    s = torch.empty((256, 5), dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    with pytest.raises(RuntimeError, match="multiple of 128"):
        L.call("fsb_quantize_w4", w.data_ptr(), 640, 256, 520, q.data_ptr(), s.data_ptr(), st)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        L.call("fsb_quantize_w4", w.data_ptr(), 640, 252, 640, q.data_ptr(), s.data_ptr(), st)
    with pytest.raises(RuntimeError, match="ldw"):
        L.call("fsb_quantize_w4", w.data_ptr(), 512, 256, 640, q.data_ptr(), s.data_ptr(), st)


# ---- GEMM ----------------------------------------------------------------------------------------------------------------
_WHAT = {}


def _weights(n, k):
    """(q, s, W^ fp64 on the device) for a seeded [n, k] weight; W^ is rebuilt by the numpy restatement from q and s."""
    if (n, k) not in _WHAT:
        g =torch.Generator(device="cuda").manual_seed(n * 7 + k)
        w = (torch.randn((n, k), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
        q, s = ops.quantize_w4(w)
        sn = s.float().cpu().numpy()
        wh = torch.from_numpy(R.dequantize(R.unpack(q.cpu().numpy()), sn)).cuda().double()
        _WHAT[(n, k)] = (q, s, wh)
    return _WHAT[(n, k)]


def _check_bound(d, a, wh):
    k = a.shape[1]
    ad = a.double()
    ref = ad @ wh.t()
    mag = ad.abs() @ wh.abs().t()
    err = (d.double() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + k * 2.0 ** -23 * mag
    assert bool((err <= bound).all()), float((err - bound).max())


# ragged n (200: a partial 128-row tile and a half 16-row slice), small shapes, and the four Ziya-13B projections
SHAPES = [(256, 512), (200, 384), (1032, 256), (15360, 5120), (5120, 5120), (27648, 5120), (5120, 13824)]


@pytest.mark.parametrize("m", [1, 3, 8, 17, 32, 64, 257, 2048])
@pytest.mark.parametrize("nk", SHAPES, ids=[f"n{n}k{k}" for n, k in SHAPES])
def test_gemm_w4a16_against_fp64(m, nk):
    n, k = nk
    q, s, wh = _weights(n, k)
    g = torch.Generator(device="cuda").manual_seed(m * 31 + n)
    lda = k + 64 if m % 2 else k                                                   # odd m: strided A (lda > k)
    a = torch.randn((m, lda), generator=g, device="cuda").to(torch.bfloat16)[:, :k]
    ldd = n + 24
    buf = torch.full((m + 5, ldd), float("nan"), dtype=torch.bfloat16, device="cuda")
    d = ops.gemm_w4a16(a, q, s, out=buf[:m, :n])                                   # strided D with a NaN sentinel
    torch.cuda.synchronize()
    assert not torch.isnan(d.float()).any()
    assert torch.isnan(buf[m:].float()).all() and torch.isnan(buf[:, n:].float()).all()
    _check_bound(d, a, wh)
    again = ops.gemm_w4a16(a, q, s)
    assert torch.equal(again, d)


@pytest.mark.parametrize("m", [1, 8, 32, 300])
def test_gemm_w4a16_graph_replay_equals_eager(m):
    n, k = 5120, 13824                       # Ziya w2: the decode calls split K
    q, s, wh = _weights(n, k)
    a = torch.randn((m, k), generator=torch.Generator(device="cuda").manual_seed(5), device="cuda").to(torch.bfloat16)
    if m <= 32:
        assert L.load().fsb_gemm_w4a16_workspace_bytes(m, n, k) > 0
    eager = ops.gemm_w4a16(a, q, s)
    out = torch.empty_like(eager)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.gemm_w4a16(a, q, s, out=out)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    _check_bound(eager, a, wh)


def test_gemm_w4a16_rejects_malformed_inputs():
    n, k, m = 256, 512, 8
    q, s, _ = _weights(n, k)
    a = torch.randn((m, k), device="cuda").to(torch.bfloat16)
    d = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def raw(m_=m, n_=n, k_=k, a_=a, lda=k, d_=d, ldd=n, ws=None, wsb=0):
        L.call("fsb_gemm_w4a16", m_, n_, k_, a_.data_ptr(), lda, q.data_ptr(), s.data_ptr(), d_.data_ptr(), ldd, ws, wsb, st)

    with pytest.raises(RuntimeError, match="multiple of 128"):
        raw(k_=496)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        raw(n_=252)
    flat = torch.zeros(m * k + 8, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="aligned"):
        ops.gemm_w4a16(flat[1:1 + m * k].view(m, k), q, s)                  # 2-byte misaligned A
    with pytest.raises(RuntimeError, match="lda"):
        ops.gemm_w4a16(torch.zeros((m, k + 4), dtype=torch.bfloat16, device="cuda")[:, :k], q, s)
    with pytest.raises(RuntimeError, match="ldd"):
        ops.gemm_w4a16(a, q, s, out=torch.zeros((m, n + 4), dtype=torch.bfloat16, device="cuda")[:, :n])
    with pytest.raises(RuntimeError):
        ops.gemm_w4a16(a, q.view(torch.int8), s)
    with pytest.raises(RuntimeError):
        ops.gemm_w4a16(a, q, s.float())
    # a call that splits K needs its workspace
    q2, s2, _ = _weights(5120, 5120)
    assert L.load().fsb_gemm_w4a16_workspace_bytes(1, 5120, 5120) > 0
    a2 = torch.randn((1, 5120), device="cuda").to(torch.bfloat16)
    d2 = torch.empty((1, 5120), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="workspace"):
        L.call("fsb_gemm_w4a16", 1, 5120, 5120, a2.data_ptr(), 5120, q2.data_ptr(), s2.data_ptr(), d2.data_ptr(), 5120,
               None, 0, st)


# ---- model -------------------------------------------------------------------------------------------------------------
def _cfg(h=256, nh=4, nl=2):
    return SimpleNamespace(vocab_size=V, hidden_size=h, num_hidden_layers=nl, num_attention_heads=nh, rms_norm_epsilon=1e-6,
                           max_position_embeddings=2048, rotary_emb_base=10000, llama_mlp_multiple_of=256)


def _dequantised(sd):
    """The oracle's weights with every projection replaced by W^."""
    out = dict(sd)
    for k, v in sd.items():
        if any(k.endswith(p) for p in PROJ):
            q, s = R.quantize(v.float().numpy())
            out[k] = torch.from_numpy(R.dequantize(q, s))
    return out


@pytest.mark.parametrize("nh", [4, 2], ids=["hd64", "hd128"])
def test_int4_model_matches_the_dequantised_oracle(nh):
    h, nl = 256, 2
    sd = O.make_weights(V, h, nl, seed=3)
    m = LlamaForCausalLM(_cfg(h, nh, nl), device="cuda", load_in_4bit=True)
    m.load_reference_state_dict(sd)
    assert m.flat.grads is None and m.weight_format == "int4" and m.load_in_4bit and not m.load_in_8bit
    q, s = m._w4[1]["qkv"]
    _check_quantized(q, s, sd["llama.layers.1.attention.query_key_value.weight"].float().numpy())
    q13, s13 = m._w4[0]["w13"]                                          # w1 | w3: one operand, w1 in the upper half
    w13 = torch.cat([sd["llama.layers.0.mlp.w1.weight"], sd["llama.layers.0.mlp.w3.weight"]]).float().numpy()
    _check_quantized(q13, s13, w13)
    sd4 = _dequantised(sd)
    batch = O.make_batch(V, 2, 48, seed=11)
    with torch.no_grad():
        out = m(input_ids=batch["input_ids"].cuda(), labels=batch["labels"].cuda())
    ref_loss, ref = O.forward(sd4, batch, nh)
    got = out.logits.float().cpu()
    tol = 4 * 2.0 ** -8 * float(ref.abs().max())
    assert float((got - ref).abs().max()) <= tol
    assert abs(out.loss.item() - ref_loss.item()) < 2e-2

    # greedy generate with left padding: on every step where the oracle is decisive, its argmax is the generated token
    B, S0, new = 3, 20, 10
    g = torch.Generator().manual_seed(12)
    ids = torch.randint(4, V, (B, S0), generator=g)
    mask = torch.ones_like(ids)
    for b in range(1, B):
        ids[b, :4 * b], mask[b, :4 * b] = 0, 0
    seqs = m.generate(ids.cuda(), attention_mask=mask.cuda(), max_new_tokens=new).cpu()
    checked = 0
    for b in range(B):
        real = seqs[b, S0 - int(mask[b].sum()):]                        # the row's tokens without its left padding
        for t in range(new):
            ctx = real[:len(real) - new + t]
            _, lg = O.forward(sd4, {"input_ids": ctx[None], "position_ids": torch.arange(len(ctx))[None]}, nh)
            top = lg[0, -1].topk(2).values
            if float(top[0] - top[1]) > 2 * tol:
                assert int(lg[0, -1].argmax()) == int(real[len(ctx)]), (b, t)
                checked += 1
    assert checked >= new


def _left_padded(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(4, V, (B, S), generator=g)
    mask = torch.ones_like(ids)
    for b in range(1, B):
        n = (5 * b) % (S - 4)
        ids[b, :n], mask[b, :n] = 0, 0
    return ids.cuda(), mask.cuda()


# LLaMA's generate is greedy or sampling (no beam search); num_return_sequences repeats each prompt in place
@pytest.mark.parametrize("kw", [dict(do_sample=False),
                                dict(do_sample=True, top_p=0.9, top_k=50, repetition_penalty=1.1, temperature=0.8,
                                     eos_token_id=2, pad_token_id=2),
                                dict(do_sample=True, top_p=0.9, num_return_sequences=3)],
                         ids=["greedy", "sampling", "sampling_nrs3"])
def test_int4_generate_graph_equals_eager(kw, monkeypatch):
    m = LlamaForCausalLM(_cfg(nh=2), device="cuda", seed=0, load_in_4bit=True)
    ids, mask = _left_padded(3, 21, seed=6)
    out = []
    for flag in ("0", "1"):
        monkeypatch.setenv("FSB_GENERATE_GRAPH", flag)
        g = torch.Generator(device="cuda").manual_seed(0)
        out.append(m.generate(ids, attention_mask=mask, max_length=21 + 20, generator=g, **kw))
    assert out[0].shape[0] == 3 * kw.get("num_return_sequences", 1)
    assert torch.equal(out[0], out[1])


def test_int4_footprint_is_below_int8():
    m4 = LlamaForCausalLM(_cfg(nh=2), device="cuda", seed=0, load_in_4bit=True)
    m8 = LlamaForCausalLM(_cfg(nh=2), device="cuda", seed=0, load_in_8bit=True)
    proj4 = sum(q.numel() + 2 * s.numel() for w4 in m4._w4 for q, s in w4.values())
    proj8 = sum(q.numel() + 4 * s.numel() for w8 in m8._w8 for q, s in w8.values())
    assert m8.get_memory_footprint() - m4.get_memory_footprint() == proj8 - proj4 > 0


# ---- loading -------------------------------------------------------------------------------------------------------------
def _save_tiny(path, sharded):
    import json
    from fengshen.models.llama.configuration_llama import LlamaConfig
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    cfg = LlamaConfig(vocab_size=V, hidden_size=256, num_hidden_layers=3, num_attention_heads=4, rms_norm_epsilon=1e-6)
    m = Compat(cfg, device="cuda", seed=7)
    m.save_pretrained(str(path))
    if sharded:   # the HF sharded layout: pytorch_model-0000i-of-0000n.bin + pytorch_model.bin.index.json
        sd = torch.load(os.path.join(path, "pytorch_model.bin"), weights_only=True)
        keys = sorted(sd)
        parts = [keys[i::3] for i in range(3)]
        wmap = {}
        for i, ks in enumerate(parts):
            fn = f"pytorch_model-{i + 1:05d}-of-00003.bin"
            torch.save({k: sd[k] for k in ks}, os.path.join(path, fn))
            wmap.update({k: fn for k in ks})
        with open(os.path.join(path, "pytorch_model.bin.index.json"), "w") as f:
            json.dump({"metadata": {}, "weight_map": wmap}, f)
        os.remove(os.path.join(path, "pytorch_model.bin"))
    return m


@pytest.mark.parametrize("sharded", [False, True], ids=["single", "sharded"])
def test_from_pretrained_load_in_4bit(tmp_path, sharded):
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    m16 = _save_tiny(tmp_path, sharded)
    want = []
    for i, lyr in enumerate(m16.llama.layers):                         # in-memory quantisation of the same weights
        want.append({"qkv": ops.quantize_w4(lyr.attention.query_key_value.weight.data),
                     "dense": ops.quantize_w4(lyr.attention.dense.weight.data),
                     "w13": ops.quantize_w4(m16._w13[i]), "w2": ops.quantize_w4(lyr.mlp.w2.weight.data)})
    head = m16.embed_out.final_linear.weight.detach().clone()
    biggest = max(v.numel() * 2 for k, v in m16.state_dict().items() if k.endswith("weight"))
    del m16
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m4 = Compat.from_pretrained(str(tmp_path), load_in_4bit=True, device_map="auto")
    torch.cuda.synchronize()
    for w4, ref in zip(m4._w4, want):
        for key in ref:
            assert torch.equal(w4[key][0], ref[key][0]) and torch.equal(w4[key][1], ref[key][1]), key
    assert torch.equal(m4.embed_out.final_linear.weight, head)
    assert m4.flat.grads is None and m4.load_in_4bit
    tensors = [m4.flat.params] + [t for w4 in m4._w4 for qs in w4.values() for t in qs]
    held = sum(t.numel() * t.element_size() for t in tensors)
    slack = (1 << 20) * (len(tensors) + len(list(m4.buffers())) + 2)
    after = torch.cuda.memory_allocated() - base
    assert after <= held + slack, (after, held)
    assert torch.cuda.max_memory_allocated() - base <= held + slack + biggest, (torch.cuda.max_memory_allocated() - base, held)


def test_from_pretrained_4bit_rejects_a_multi_device_map_and_both_flags(tmp_path):
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    _save_tiny(tmp_path, False)
    with pytest.raises(NotImplementedError, match="device"):
        Compat.from_pretrained(str(tmp_path), load_in_4bit=True, device_map={"llama.embed_in": 0, "llama.layers": 1})
    with pytest.raises(ValueError, match="load_in_4bit"):
        Compat.from_pretrained(str(tmp_path), load_in_8bit=True, load_in_4bit=True)
    with pytest.raises(ValueError, match="load_in_4bit"):
        LlamaForCausalLM(_cfg(), device="cuda", load_in_8bit=True, load_in_4bit=True)


# ---- what an int4 model refuses ----------------------------------------------------------------------------------------------
def test_int4_model_refuses_training_tp_and_export(tmp_path, monkeypatch):
    from fsb200.engine import ZeroEngine
    from fsb200.trainer import PretrainStep
    msg = r"int4 \(load_in_4bit=True\)"
    m = LlamaForCausalLM(_cfg(), device="cuda", load_in_4bit=True)
    ids = torch.randint(4, V, (2, 16), generator=torch.Generator().manual_seed(1)).cuda()
    with pytest.raises(NotImplementedError, match=msg):
        m(input_ids=ids, labels=ids)
    with pytest.raises(NotImplementedError, match=msg):
        ZeroEngine(m)
    with pytest.raises(NotImplementedError, match=msg):
        PretrainStep(m, lambda s_: 1e-3)
    with pytest.raises(NotImplementedError, match=msg):
        m.save_pretrained(str(tmp_path / "x"))
    import torch.distributed as dist
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    with pytest.raises(NotImplementedError, match=msg):
        LlamaForCausalLM(_cfg(), device="cuda", load_in_4bit=True, tp_group=object())
    monkeypatch.undo()
    from fengshen.models.llama.configuration_llama import LlamaConfig
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    c = Compat(LlamaConfig(vocab_size=V, hidden_size=256, num_hidden_layers=1, num_attention_heads=4), device="cuda",
               load_in_4bit=True)
    with pytest.raises(NotImplementedError, match=msg):
        c.save_pretrained(str(tmp_path / "y"))
    with pytest.raises(RuntimeError, match="multiples of 128"):
        LlamaForCausalLM(_cfg(h=192, nh=3), device="cuda", load_in_4bit=True)
    with torch.no_grad():                     # no-grad forward with labels is inference: loss and logits
        out = m(input_ids=ids, labels=ids)
    assert torch.isfinite(out.loss) and out.logits.shape == (2, 16, V)
