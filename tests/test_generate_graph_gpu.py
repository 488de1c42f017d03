"""GPU: the CUDA-graph decode step of `generate` (fsb200/decode_graph.py) and the two kernels that keep its position on the
device. fsb_kv_append and fsb_kv_reorder are checked against torch indexing, with NaN sentinels proving that nothing outside
the target slots is written. The graphed `generate` of GPT-2, mT5 and LLaMA must equal the same step body run eagerly
(FSB_GENERATE_GRAPH=0) bit for bit: tokens, every step's scores and the beam scores."""
import os
import sys
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fengshen-lm_b200", "compat"))

from fsb200 import lib as L  # noqa: E402
from fsb200 import ops  # noqa: E402
from fsb200.models.gpt2 import GPT2LMHeadModel  # noqa: E402
from fsb200.models.llama import LlamaForCausalLM  # noqa: E402
from fsb200.models.t5 import MT5ForConditionalGeneration  # noqa: E402

V = 512


def _bf16_randn(shape, g):
    return torch.randn(shape, generator=g, device="cuda").to(torch.bfloat16)


# ---- fsb_kv_append ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["packed", "interleaved"])
@pytest.mark.parametrize("D", [64, 128])
def test_kv_append_writes_one_slot_of_both_layouts(layout, D):
    g = torch.Generator(device="cuda").manual_seed(D)
    R, H, cap = 6, 3, 128
    nan = float("nan")
    for slot in (0, 77, cap - 1):
        if layout == "packed":     # GPT-2 / mT5: [t, {q,k,v}, head, d] into one [rows, cap, 2, heads, d] cache
            src = _bf16_randn((R, 3, H, D), g)
            kn, vn = src[:, 1], src[:, 2]
            cache = torch.full((R, cap, 2, H, D), nan, dtype=torch.bfloat16, device="cuda")
            kc, vc = cache[:, :, 0], cache[:, :, 1]
        else:                      # LLaMA: [t, head, {q,k,v}, d] into separate [rows, cap, heads, d] caches
            src = _bf16_randn((R, H, 3, D), g)
            kn, vn = src[:, :, 1], src[:, :, 2]
            kc = torch.full((R, cap, H, D), nan, dtype=torch.bfloat16, device="cuda")
            vc = torch.full((R, cap, H, D), nan, dtype=torch.bfloat16, device="cuda")
        mask = torch.zeros((R, cap), dtype=torch.uint8, device="cuda")
        kv_len = torch.tensor([slot + 1], dtype=torch.int32, device="cuda")
        ops.kv_append(kn, vn, kc, vc, kv_len, kv_mask=mask)
        assert torch.equal(kc[:, slot], kn) and torch.equal(vc[:, slot], vn)
        others = [s for s in range(cap) if s != slot]
        assert torch.isnan(kc[:, others].float()).all() and torch.isnan(vc[:, others].float()).all()
        want = torch.zeros_like(mask)
        want[:, slot] = 1
        assert torch.equal(mask, want)
        ops.kv_append(kn, vn, kc, vc, kv_len)          # without a mask: the mask is not touched
        assert torch.equal(mask, want)


def test_kv_append_outside_the_cache_writes_nothing():
    g = torch.Generator(device="cuda").manual_seed(1)
    R, H, D, cap = 4, 2, 64, 64
    src = _bf16_randn((R, 3, H, D), g)
    cache = torch.full((R, cap, 2, H, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    mask = torch.zeros((R, cap), dtype=torch.uint8, device="cuda")
    for n in (0, cap + 1, -5):
        ops.kv_append(src[:, 1], src[:, 2], cache[:, :, 0], cache[:, :, 1],
                      torch.tensor([n], dtype=torch.int32, device="cuda"), kv_mask=mask)
    torch.cuda.synchronize()
    assert torch.isnan(cache.float()).all() and not mask.any()


# ---- fsb_kv_reorder --------------------------------------------------------------------------------------------------
def test_kv_reorder_gathers_the_live_prefix_of_every_layer_in_one_launch(monkeypatch):
    g = torch.Generator(device="cuda").manual_seed(2)
    Ly, R, cap, H, D = 3, 6, 192, 4, 64
    src = _bf16_randn((Ly, R, cap, 2, H, D), g)
    calls = []
    real = L.call
    monkeypatch.setattr(L, "call", lambda name, *a, **k: (calls.append(name), real(name, *a, **k))[1])
    for index in ([5, 0, 0, 3, 3, 3], [1, 1, 2, 2, 4, 4], [0, 1, 2, 3, 4, 5]):
        idx = torch.tensor(index, dtype=torch.int64, device="cuda")
        for n in (1, 101, cap):
            dst = torch.full_like(src, float("nan"))
            calls.clear()
            ops.kv_reorder(src, dst, idx, torch.tensor([n], dtype=torch.int32, device="cuda"))
            assert calls == ["fsb_kv_reorder"]
            assert torch.equal(dst[:, :, :n], src.index_select(1, idx)[:, :, :n])
            assert torch.isnan(dst[:, :, n:].float()).all()


# ---- graphed generate == eager generate --------------------------------------------------------------------------------
def _gpt2(seed=0):
    import transformers
    cfg = transformers.GPT2Config(vocab_size=V, n_positions=256, n_embd=256, n_layer=2, n_head=4, bos_token_id=3,
                                  eos_token_id=3, resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)
    m = GPT2LMHeadModel(cfg, device="cuda", world_size=1, seed=seed)
    with torch.no_grad():
        m.transformer.ln_f.weight.mul_(8.0)        # sharper logits: the searches take distinct paths
    return m


def _mt5(seed=0):
    import transformers
    cfg = transformers.MT5Config(vocab_size=V, d_model=256, d_kv=64, d_ff=512, num_layers=2, num_heads=4,
                                 relative_attention_num_buckets=32, dropout_rate=0.0, pad_token_id=0, eos_token_id=1,
                                 decoder_start_token_id=0)
    return MT5ForConditionalGeneration(cfg, device="cuda", world_size=1, seed=seed)


def _llama(seed=0):
    cfg = SimpleNamespace(vocab_size=V, hidden_size=256, num_hidden_layers=2, num_attention_heads=2, rms_norm_epsilon=1e-6,
                          max_position_embeddings=2048, rotary_emb_base=10000, llama_mlp_multiple_of=256)
    return LlamaForCausalLM(cfg, device="cuda", seed=seed)


def _both(monkeypatch, fn):
    """fn() with the decode step eager (FSB_GENERATE_GRAPH=0), then graphed."""
    out = []
    for flag in ("0", "1"):
        monkeypatch.setenv("FSB_GENERATE_GRAPH", flag)
        torch.manual_seed(1234)
        out.append(fn())
    return out


def _assert_same(a, b):
    if isinstance(a, torch.Tensor):
        assert torch.equal(a, b)
        return
    assert torch.equal(a.sequences, b.sequences)
    assert (a.scores is None) == (b.scores is None)
    if a.scores is not None:
        assert len(a.scores) == len(b.scores)
        for t, (x, y) in enumerate(zip(a.scores, b.scores)):
            assert torch.equal(x, y), t
    assert (a.sequences_scores is None) == (b.sequences_scores is None)
    if a.sequences_scores is not None:
        assert torch.equal(a.sequences_scores, b.sequences_scores)


def _left_padded(B, S, pad, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(4, V, (B, S), generator=g)
    mask = torch.ones_like(ids)
    for b in range(1, B):
        n = (5 * b) % (S - 4)
        ids[b, :n], mask[b, :n] = pad, 0
    return ids.cuda(), mask.cuda()


GPT2_CASES = {
    "greedy": dict(max_new_tokens=20),
    "sampling": dict(max_new_tokens=20, do_sample=True, top_k=40, top_p=0.9, repetition_penalty=1.3, temperature=0.8),
    "return_sequences": dict(max_new_tokens=16, do_sample=True, num_return_sequences=3),
    "beam3": dict(max_new_tokens=16, num_beams=3, num_return_sequences=2, length_penalty=0.7),
    "scores": dict(max_new_tokens=16, return_dict_in_generate=True, output_scores=True, repetition_penalty=1.2),
    "beam_scores": dict(max_new_tokens=16, num_beams=3, return_dict_in_generate=True, output_scores=True),
}


@pytest.mark.parametrize("case", sorted(GPT2_CASES))
def test_gpt2_graph_equals_eager(case, monkeypatch):
    m = _gpt2()
    ids = torch.randint(4, V, (3, 24), generator=torch.Generator().manual_seed(7)).cuda()
    a, b = _both(monkeypatch, lambda: m.generate(input_ids=ids, **GPT2_CASES[case]))
    _assert_same(a, b)


def test_gpt2_left_padding_graph_equals_eager(monkeypatch):
    m = _gpt2(seed=1)
    ids, mask = _left_padded(4, 30, 3, seed=8)
    for kw in (dict(max_new_tokens=18, return_dict_in_generate=True, output_scores=True),
               dict(max_new_tokens=12, num_beams=3, return_dict_in_generate=True, output_scores=True)):
        a, b = _both(monkeypatch, lambda: m.generate(input_ids=ids, attention_mask=mask, **kw))
        _assert_same(a, b)


@pytest.mark.parametrize("kw", [dict(max_length=20), dict(max_length=16, num_beams=2, repetition_penalty=2.5),
                                dict(max_length=16, num_beams=3, return_dict_in_generate=True, output_scores=True),
                                dict(max_length=14, do_sample=True, top_k=20)],
                         ids=["greedy", "beam2", "beam3_scores", "sampling"])
def test_mt5_graph_equals_eager_with_padded_encoder_rows(kw, monkeypatch):
    m = _mt5()
    ids, mask = _left_padded(3, 29, 0, seed=5)
    mask, ids = mask.flip(1), ids.flip(1)           # right-padded encoder rows, as the summary recipe feeds them
    a, b = _both(monkeypatch, lambda: m.generate(input_ids=ids, attention_mask=mask, **kw))
    _assert_same(a, b)


@pytest.mark.parametrize("kw", [dict(do_sample=False), dict(do_sample=True, top_p=0.9, top_k=50, repetition_penalty=1.1,
                                                            temperature=0.8, eos_token_id=2, pad_token_id=2)],
                         ids=["greedy", "sampling"])
def test_llama_graph_equals_eager_with_left_padding(kw, monkeypatch):
    m = _llama()
    ids, mask = _left_padded(3, 21, 0, seed=6)

    def run():
        g = torch.Generator(device="cuda").manual_seed(0)
        return m.generate(ids, attention_mask=mask, max_length=21 + 20, generator=g, **kw)
    a, b = _both(monkeypatch, run)
    _assert_same(a, b)


# ---- the graph is really used ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gpt2", "mt5", "llama"])
def test_host_calls_do_not_grow_with_new_tokens(kind, monkeypatch):
    """Graphed: 10 and 30 new tokens issue the same number of host `fsb_*` calls (prefill, the eager warm-up step and the
    capture). Eager: the count grows by the per-step calls of 20 more steps."""
    n = {"calls": 0}
    real = L.call

    def counted(name, *a, **k):
        n["calls"] += 1
        return real(name, *a, **k)

    monkeypatch.setattr(L, "call", counted)
    m = {"gpt2": _gpt2, "mt5": _mt5, "llama": _llama}[kind]()
    ids = torch.randint(4, V, (2, 16), generator=torch.Generator().manual_seed(3)).cuda()
    nl = 2

    def calls(new):
        n["calls"] = 0
        if kind == "llama":
            m.generate(ids, max_length=16 + new, eos_token_id=None)
        elif kind == "mt5":
            m.generate(input_ids=ids, max_length=1 + new, eos_token_id=V)
        else:
            m.generate(input_ids=ids, max_new_tokens=new, eos_token_id=V)
        return n["calls"]

    counts = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("FSB_GENERATE_GRAPH", flag)
        counts[flag] = (calls(10), calls(30))
    assert counts["1"][0] == counts["1"][1], counts
    per_step = (counts["0"][1] - counts["0"][0]) / 20
    assert per_step >= 6 * nl, counts          # at least the layer kernels of every eager step
    assert counts["1"][1] < counts["0"][1] - 15 * per_step


@pytest.mark.parametrize("kind", ["gpt2", "mt5", "llama"])
def test_generate_releases_its_memory_on_return(kind, monkeypatch):
    """The caches (the beam twin included), the static buffers and the graphs of a `generate` call are freed when it
    returns, by reference counting alone: no reference cycle holds them until the garbage collector runs."""
    import gc
    m = {"gpt2": _gpt2, "mt5": _mt5, "llama": _llama}[kind]()
    ids = torch.randint(4, V, (2, 16), generator=torch.Generator().manual_seed(3)).cuda()
    if kind == "llama":
        gen = lambda: m.generate(ids, max_length=16 + 8)                                          # noqa: E731
    else:
        gen = lambda: m.generate(input_ids=ids, max_new_tokens=8, num_beams=2, eos_token_id=V)   # noqa: E731
    monkeypatch.setenv("FSB_GENERATE_GRAPH", "1")
    gen()                              # workspaces and tables that persist across calls
    torch.cuda.synchronize()
    gc.collect()
    gc.disable()
    try:
        base = torch.cuda.memory_allocated()
        gen()
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == base
    finally:
        gc.enable()


def test_parameters_updated_between_calls_are_seen(monkeypatch):
    """A training step between two generate calls: the graphed decode reads the updated weights (it equals the eager decode
    after the step, and differs from the decode before it)."""
    from fsb200.trainer import PretrainStep
    m = _gpt2()
    st = PretrainStep(m, lambda s_: 1e-2, lr=1e-2, weight_decay=0.0)
    ids = torch.randint(4, V, (3, 24), generator=torch.Generator().manual_seed(9)).cuda()
    kw = dict(max_new_tokens=12, return_dict_in_generate=True, output_scores=True)
    monkeypatch.setenv("FSB_GENERATE_GRAPH", "1")
    before = m.generate(input_ids=ids, **kw)
    batch = torch.randint(4, V, (4, 32), generator=torch.Generator().manual_seed(10))
    st.step([{"input_ids": batch, "labels": batch}])
    a, b = _both(monkeypatch, lambda: m.generate(input_ids=ids, **kw))
    _assert_same(a, b)
    assert not torch.equal(torch.stack(before.scores), torch.stack(b.scores))
