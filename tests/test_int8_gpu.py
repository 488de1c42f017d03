"""GPU: int8 weight-only LLaMA inference. The quantiser (fsb_quantize_w8) against a numpy float32 restatement of its formula,
bit for bit; the W8A16 GEMM (fsb_gemm_w8a16) against fp64 with the error bound its fp32 accumulation allows, NaN sentinels,
determinism and graph capture; the `load_in_8bit` LLaMA against the CPU oracle with every projection replaced by q * s;
graphed against eager generate; shard-by-shard loading and its memory; and the paths an int8 model refuses."""
import json
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

import int8_ref  # noqa: E402
import llama_oracle as O  # noqa: E402
from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402

V = 512
PROJ = ("attention.query_key_value.weight", "attention.dense.weight", "mlp.w1.weight", "mlp.w3.weight", "mlp.w2.weight")


np_quantize = int8_ref.quantize


def _bf16(x):
    return torch.as_tensor(x, dtype=torch.float32).to(torch.bfloat16)


# ---- quantiser ---------------------------------------------------------------------------------------------------------
def test_quantize_matches_numpy_bit_for_bit():
    g = torch.Generator().manual_seed(0)
    k = 1040
    rows = [torch.randn(k, generator=g) * mag for mag in (2.0 ** -60, 1e-3, 1.0, 37.0, 1e3, 2.0 ** 60)]
    rows.append(torch.zeros(k))                                           # all-zero row
    out = torch.randn(k, generator=g) * 1e-2
    out[517] = 900.0
    rows.append(out)                                                      # one outlier
    half = torch.zeros(k)                                                 # s = 127 / 127 = 1: exact half-steps
    half[:9] = torch.tensor([127.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5, -125.5])
    rows.append(half)
    rows.append(-half)
    w = _bf16(torch.stack(rows))
    wide = torch.full((w.shape[0], k + 72), float("nan"), dtype=torch.bfloat16)
    wide[:, :k] = w
    for src in (w.cuda(), wide.cuda()[:, :k]):                            # contiguous and strided (ldw > k)
        q, s = ops.quantize_w8(src)
        qn, sn = np_quantize(w.float().numpy())
        assert np.array_equal(q.cpu().numpy(), qn)
        assert np.array_equal(s.cpu().numpy().view(np.int32), sn.view(np.int32))
    assert q[-2, :9].tolist() == [127, 0, 2, 2, 0, -2, -2, 126, -126]    # ties to even
    assert s[6].item() == 0.0 and not q[6].any()


# ---- GEMM ----------------------------------------------------------------------------------------------------------------
def _operands(m, n, k, seed, lda=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn((n, k), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    q, s = ops.quantize_w8(w)
    lda = k if lda is None else lda
    abuf = torch.randn((m, lda), generator=g, device="cuda").to(torch.bfloat16)
    return abuf[:, :k], q, s


def _check_bound(d, a, q, s):
    k = a.shape[1]
    ad, qd, sd = a.double(), q.double(), s.double()
    ref = (ad @ qd.t()) * sd
    mag = (ad.abs() @ qd.abs().t()) * sd
    err = (d.double() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + k * 2.0 ** -23 * mag
    assert bool((err <= bound).all()), float((err - bound).max())


SHAPES = [(256, 512), (200, 48), (1032, 272), (5120, 5120)]


@pytest.mark.parametrize("m", [1, 3, 8, 17, 64, 257, 2048])
@pytest.mark.parametrize("nk", SHAPES, ids=[f"n{n}k{k}" for n, k in SHAPES])
def test_gemm_w8a16_against_fp64(m, nk):
    n, k = nk
    a, q, s = _operands(m, n, k, seed=m * 31 + n, lda=k + 64 if m % 2 else k)   # odd m: strided A (lda > k)
    ldd = n + 24
    buf = torch.full((m + 5, ldd), float("nan"), dtype=torch.bfloat16, device="cuda")
    d = ops.gemm_w8a16(a, q, s, out=buf[:m, :n])                                   # strided D with a NaN sentinel
    torch.cuda.synchronize()
    assert not torch.isnan(d.float()).any()
    assert torch.isnan(buf[m:].float()).all() and torch.isnan(buf[:, n:].float()).all()
    _check_bound(d, a, q, s)
    again = ops.gemm_w8a16(a, q, s)
    assert torch.equal(again, d)


@pytest.mark.parametrize("m", [1, 8, 32, 300])
def test_gemm_w8a16_graph_replay_equals_eager(m):
    n, k = 5120, 13824                       # Ziya w2: the decode calls split K
    a, q, s = _operands(m, n, k, seed=5)
    eager = ops.gemm_w8a16(a, q, s)
    out = torch.empty_like(eager)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.gemm_w8a16(a, q, s, out=out)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    _check_bound(eager, a, q, s)


def test_gemm_w8a16_rejects_malformed_inputs():
    a, q, s = _operands(8, 256, 512, seed=1)
    with pytest.raises(RuntimeError, match="multiple of 16"):
        qq, ss = ops.quantize_w8(torch.zeros((256, 520), dtype=torch.bfloat16, device="cuda"))
        ops.gemm_w8a16(torch.zeros((8, 520), dtype=torch.bfloat16, device="cuda"), qq, ss)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        qq, ss = ops.quantize_w8(torch.zeros((252, 512), dtype=torch.bfloat16, device="cuda"))
        ops.gemm_w8a16(a, qq, ss)
    flat = torch.zeros(8 * 512 + 8, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="aligned"):
        ops.gemm_w8a16(flat[1:1 + 8 * 512].view(8, 512), q, s)             # 2-byte misaligned A
    with pytest.raises(RuntimeError, match="lda"):
        ops.gemm_w8a16(torch.zeros((8, 516), dtype=torch.bfloat16, device="cuda")[:, :512], q, s)
    with pytest.raises(RuntimeError, match="ldd"):
        ops.gemm_w8a16(a, q, s, out=torch.zeros((8, 260), dtype=torch.bfloat16, device="cuda")[:, :256])
    with pytest.raises(RuntimeError):
        ops.gemm_w8a16(a, q.to(torch.bfloat16), s)
    # a call that splits K needs its workspace
    a2, q2, s2 = _operands(1, 5120, 5120, seed=2)
    assert L.load().fsb_gemm_w8a16_workspace_bytes(1, 5120, 5120) > 0
    d = torch.empty((1, 5120), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="workspace"):
        L.call("fsb_gemm_w8a16", 1, 5120, 5120, a2.data_ptr(), 5120, q2.data_ptr(), s2.data_ptr(), d.data_ptr(), 5120,
               None, 0, torch.cuda.current_stream().cuda_stream)


# ---- model -------------------------------------------------------------------------------------------------------------
def _cfg(h=256, nh=4, nl=2):
    return SimpleNamespace(vocab_size=V, hidden_size=h, num_hidden_layers=nl, num_attention_heads=nh, rms_norm_epsilon=1e-6,
                           max_position_embeddings=2048, rotary_emb_base=10000, llama_mlp_multiple_of=256)


def _dequantised(sd):
    """The oracle's weights with every projection replaced by q * s."""
    out = dict(sd)
    for k, v in sd.items():
        if any(k.endswith(p) for p in PROJ):
            q, s = np_quantize(v.numpy())
            out[k] = torch.from_numpy(q.astype(np.float32) * s[:, None])
    return out


@pytest.mark.parametrize("nh", [4, 2], ids=["hd64", "hd128"])
def test_int8_model_matches_the_dequantised_oracle(nh):
    h, nl = 256, 2
    sd = O.make_weights(V, h, nl, seed=3)
    m = LlamaForCausalLM(_cfg(h, nh, nl), device="cuda", load_in_8bit=True)
    m.load_reference_state_dict(sd)
    assert m.flat.grads is None
    q, s = m._w8[1]["qkv"]
    qn, sn = np_quantize(sd["llama.layers.1.attention.query_key_value.weight"].numpy())
    assert np.array_equal(q.cpu().numpy(), qn) and np.array_equal(s.cpu().numpy(), sn)
    sd8 = _dequantised(sd)
    batch = O.make_batch(V, 2, 48, seed=11)
    with torch.no_grad():
        out = m(input_ids=batch["input_ids"].cuda(), labels=batch["labels"].cuda())
    ref_loss, ref = O.forward(sd8, batch, nh)
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
            _, lg = O.forward(sd8, {"input_ids": ctx[None], "position_ids": torch.arange(len(ctx))[None]}, nh)
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


@pytest.mark.parametrize("kw", [dict(do_sample=False), dict(do_sample=True, top_p=0.9, top_k=50, repetition_penalty=1.1,
                                                            temperature=0.8, eos_token_id=2, pad_token_id=2)],
                         ids=["greedy", "sampling"])
def test_int8_generate_graph_equals_eager(kw, monkeypatch):
    m = LlamaForCausalLM(_cfg(nh=2), device="cuda", seed=0, load_in_8bit=True)
    ids, mask = _left_padded(3, 21, seed=6)
    out = []
    for flag in ("0", "1"):
        monkeypatch.setenv("FSB_GENERATE_GRAPH", flag)
        g = torch.Generator(device="cuda").manual_seed(0)
        out.append(m.generate(ids, attention_mask=mask, max_length=21 + 20, generator=g, **kw))
    assert torch.equal(out[0], out[1])


def test_int8_generate_host_calls_do_not_grow_with_new_tokens(monkeypatch):
    n = {"calls": 0}
    real = L.call

    def counted(name, *a, **k):
        n["calls"] += 1
        return real(name, *a, **k)

    monkeypatch.setattr(L, "call", counted)
    m = LlamaForCausalLM(_cfg(nh=2), device="cuda", seed=0, load_in_8bit=True)
    ids = torch.randint(4, V, (2, 16), generator=torch.Generator().manual_seed(3)).cuda()

    def calls(new):
        n["calls"] = 0
        m.generate(ids, max_length=16 + new, eos_token_id=None)
        return n["calls"]

    counts = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("FSB_GENERATE_GRAPH", flag)
        counts[flag] = (calls(10), calls(30))
    assert counts["1"][0] == counts["1"][1], counts
    assert counts["0"][1] > counts["0"][0], counts


def test_int8_num_return_sequences_and_footprint():
    m8 = LlamaForCausalLM(_cfg(nh=2), device="cuda", seed=0, load_in_8bit=True)
    m16 = LlamaForCausalLM(_cfg(nh=2), device="cuda", seed=0)
    assert m8.get_memory_footprint() < m16.get_memory_footprint() / 2
    ids = torch.randint(4, V, (2, 12), generator=torch.Generator().manual_seed(4)).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    out = m8.generate(ids, max_new_tokens=6, do_sample=True, top_p=0.9, num_return_sequences=3, generator=g)
    assert out.shape == (6, 18)


# ---- loading -------------------------------------------------------------------------------------------------------------
def _save_tiny(path, sharded):
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
def test_from_pretrained_load_in_8bit(tmp_path, sharded):
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    m16 = _save_tiny(tmp_path, sharded)
    want = []
    for i, lyr in enumerate(m16.llama.layers):
        want.append({"qkv": ops.quantize_w8(lyr.attention.query_key_value.weight.data),
                     "dense": ops.quantize_w8(lyr.attention.dense.weight.data),
                     "w13": ops.quantize_w8(m16._w13[i]), "w2": ops.quantize_w8(lyr.mlp.w2.weight.data)})
    head = m16.embed_out.final_linear.weight.detach().clone()
    biggest = max(v.numel() * 2 for k, v in m16.state_dict().items() if k.endswith("weight"))
    del m16
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m8 = Compat.from_pretrained(str(tmp_path), load_in_8bit=True, device_map="auto")
    torch.cuda.synchronize()
    for w8, ref in zip(m8._w8, want):
        for key in ref:
            assert torch.equal(w8[key][0], ref[key][0]) and torch.equal(w8[key][1], ref[key][1]), key
    assert torch.equal(m8.embed_out.final_linear.weight, head)
    assert m8.flat.grads is None
    tensors = [m8.flat.params] + [t for w8 in m8._w8 for qs in w8.values() for t in qs]
    held = sum(t.numel() * t.element_size() for t in tensors)
    slack = (1 << 20) * (len(tensors) + len(list(m8.buffers())) + 2)
    after = torch.cuda.memory_allocated() - base
    assert after <= held + slack, (after, held)
    assert torch.cuda.max_memory_allocated() - base <= held + slack + biggest, (torch.cuda.max_memory_allocated() - base, held)


def test_from_pretrained_rejects_a_multi_device_map(tmp_path):
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    _save_tiny(tmp_path, False)
    with pytest.raises(NotImplementedError, match="device"):
        Compat.from_pretrained(str(tmp_path), load_in_8bit=True, device_map={"llama.embed_in": 0, "llama.layers": 1})


# ---- what an int8 model refuses ----------------------------------------------------------------------------------------------
def test_int8_model_refuses_training_tp_and_export(tmp_path, monkeypatch):
    from fsb200.engine import ZeroEngine
    from fsb200.trainer import PretrainStep
    m = LlamaForCausalLM(_cfg(), device="cuda", load_in_8bit=True)
    ids = torch.randint(4, V, (2, 16), generator=torch.Generator().manual_seed(1)).cuda()
    with pytest.raises(NotImplementedError, match="int8"):
        m(input_ids=ids, labels=ids)
    with pytest.raises(NotImplementedError, match="int8"):
        ZeroEngine(m)
    with pytest.raises(NotImplementedError, match="int8"):
        PretrainStep(m, lambda s_: 1e-3)
    with pytest.raises(NotImplementedError, match="int8"):
        m.save_pretrained(str(tmp_path / "x"))
    import torch.distributed as dist
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    with pytest.raises(NotImplementedError, match="int8"):
        LlamaForCausalLM(_cfg(), device="cuda", load_in_8bit=True, tp_group=object())
    monkeypatch.undo()
    from fengshen.models.llama.configuration_llama import LlamaConfig
    from fengshen.models.llama.modeling_llama import LlamaForCausalLM as Compat
    c = Compat(LlamaConfig(vocab_size=V, hidden_size=256, num_hidden_layers=1, num_attention_heads=4), device="cuda",
               load_in_8bit=True)
    with pytest.raises(NotImplementedError, match="int8"):
        c.save_pretrained(str(tmp_path / "y"))
    with torch.no_grad():                     # no-grad forward with labels is inference: loss and logits
        out = m(input_ids=ids, labels=ids)
    assert torch.isfinite(out.loss) and out.logits.shape == (2, 16, V)
